"""Env-id sharding across the GPUs of one box (one process per GPU).

The batched step path shards naturally: envs are independent (own mt19937, own state), so
rank r of G owns the contiguous global ids [offset, offset + count) and seeds them with
`seed + global_env_id` exactly as a single pool would (envpool/core/env.h:101-111) -- results
do not depend on G.  The one exchange step of the path is an all-gather of the output
columns, which reassembles the full `[num_envs, ...]` batch on every rank.  Two transports:

* the engine's own peer exchange (csrc/exchange.cuh): the step writes into this rank's slice
  of a ring of gather slots that every peer maps through CUDA IPC, a copy kernel behind it stores
  the columns a peer cannot derive (env keys, reward, one packed word) into all peers over
  NVLink and raises sequence flags; the receiver re-expands the rest --
  `enable_peer_exchange()`, `reset_exchange()`, `step_exchange(actions)`;
* `torch.distributed` all-gather (NCCL on GPUs; gloo on CPU tensors in the host-logic
  tests) -- `all_gather()`; also the cross-check of the first.

    pool = ShardedPool("CartPole-v1", num_envs=1 << 20)         # inside torchrun
    pool.enable_peer_exchange()
    full = pool.reset_exchange()                # {key: [world, n_local, ...]} on every rank
    full = pool.step_exchange(local_actions)
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

# The task kwargs a shard hands to its pool, by engine task (the keys PoolBase::Create in
# csrc/py_module.cc maps into epb_config), plus the ones that change no output column.  An
# explicitly passed kwarg outside this list is refused: dropping it would run the shard with
# the default while the caller believes otherwise.
_COMMON_KWARGS = ("max_episode_steps", "reward_threshold", "base_path")
_TASK_KWARGS = {
    "FrozenLake": ("size",), "Pendulum": ("version",), "CliffWalking": ("is_slippery",),
    "Blackjack": ("natural", "sab"),
    "HalfCheetah": ("frame_skip", "ctrl_cost_weight", "forward_reward_weight",
                    "reset_noise_scale", "post_constraint", "gymnasium_v5_render_camera"),
    "Go": ("komi", "max_terminal_steps"),
}
# ... and of every multi-player kind: its registration's `task` and max_num_players
_PLAYER_KWARGS = ("task", "max_num_players")


def shard_range(num_envs: int, rank: int, world: int) -> Tuple[int, int]:
    """(global id of the first local env, number of local envs) for `rank` of `world`.
    Contiguous blocks; the all-gather needs equal shards, so num_envs % world must be 0."""
    if world <= 0 or not 0 <= rank < world:
        raise ValueError(f"bad rank/world: {rank}/{world}")
    if num_envs % world != 0:
        raise ValueError(f"num_envs={num_envs} is not divisible by world_size={world}")
    count = num_envs // world
    return rank * count, count


def all_gather_columns(local: Dict[str, "object"], full: Optional[Dict[str, "object"]] = None,
                       group=None) -> Dict[str, "object"]:
    """All-gather every column of `local` ({key: tensor [n_local, ...]}) into `full`
    ({key: tensor [world * n_local, ...]}, allocated when None).  Rank r's rows land at
    [r * n_local, (r + 1) * n_local): global env-id order."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    if full is None:
        full = {k: torch.empty((world * v.shape[0],) + tuple(v.shape[1:]), dtype=v.dtype,
                               device=v.device) for k, v in local.items()}
    for k, v in local.items():
        src = v if v.is_contiguous() else v.contiguous()
        if src.dtype == torch.bool:  # gloo/nccl move bytes; bool is reinterpreted as uint8
            dist.all_gather_into_tensor(full[k].view(torch.uint8), src.view(torch.uint8),
                                        group=group)
        else:
            dist.all_gather_into_tensor(full[k], src, group=group)
    return full


def all_gather_packed(local_slab, full_slab=None, group=None):
    """ONE collective for the whole step: all-gather the packed output slab (every column of
    this rank, `slab_bytes` uint8) into `[world, slab_bytes]`.  Column k of rank r then sits
    at `full[r, off_k : off_k + n_local*row_bytes]`; `packed_views` exposes it as a
    `[world, n_local, ...]` tensor (global env-id order along the first two dims)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    if full_slab is None:
        full_slab = torch.empty((world, local_slab.numel()), dtype=torch.uint8,
                                device=local_slab.device)
    dist.all_gather_into_tensor(full_slab, local_slab, group=group)
    return full_slab


def packed_views(full_slab, keys, n_local):
    """{key: [world, n_local, ...] strided view} into a gathered slab (zero-copy)."""
    import numpy as np
    import torch

    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    out = {}
    world = full_slab.shape[0]
    for k in keys:
        nb = k.row_bytes * n_local
        col = full_slab[:, k.offset:k.offset + nb]                 # [world, nb] uint8
        out[k.name] = col.view(tdt[k.dtype]).view((world, n_local) + tuple(k.shape))
    return out


class ShardedPool:
    """This rank's shard of a `num_envs`-wide pool plus the all-gather of its outputs."""

    def __init__(self, task_id: str, num_envs: int, seed: int = 42, group=None,
                 device: Optional[int] = None, precision: str = "f64", **task_kwargs):
        import torch
        import torch.distributed as dist

        from . import _capi
        from .registration import registry
        from . import _ensure_registered

        _ensure_registered()
        _, spec_cls, kwargs = registry.specs[task_id]
        engine_task = spec_cls.replace("EnvSpec", "").replace("Gym", "")
        players = kwargs.get("max_num_players", 1)  # as registered: the kind's players per env
        dropped = sorted(set(task_kwargs) - set(_COMMON_KWARGS) -
                         set(_TASK_KWARGS.get(engine_task, ())) -
                         set(_PLAYER_KWARGS if players > 1 else ()))
        if dropped:
            raise ValueError(f"ShardedPool({task_id!r}) cannot carry {dropped} to its shards")
        kwargs = {**kwargs, **task_kwargs}
        if kwargs.get("max_num_players", 1) != players:
            raise ValueError(f"ShardedPool({task_id!r}): max_num_players must be {players}")
        hc = {}
        if engine_task == "HalfCheetah":
            hc = dict(frame_skip=kwargs.get("frame_skip", 5),
                      ctrl_cost_weight=kwargs.get("ctrl_cost_weight", math.nan),
                      forward_reward_weight=kwargs.get("forward_reward_weight", math.nan),
                      reset_noise_scale=kwargs.get("reset_noise_scale", math.nan))
            if hc["frame_skip"] < 1:   # as make(): the reward divides by frame_skip * timestep
                raise ValueError(f"HalfCheetah: frame_skip must be >= 1, got {hc['frame_skip']}")
        go = {}
        if engine_task == "Go":  # one engine kind per board size
            engine_task = "Go{0}x{0}".format(kwargs["board_size"])
            go = dict(komi=kwargs.get("komi", 7.5),
                      max_terminal_steps=kwargs.get("max_terminal_steps", 0))
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.offset, self.count = shard_range(num_envs, self.rank, self.world)
        self.num_envs = num_envs
        if device is None:
            device = torch.cuda.current_device()
        iopt = -1
        if engine_task == "FrozenLake":
            iopt = kwargs.get("size", 4)
        elif engine_task == "Pendulum":
            iopt = kwargs.get("version", 0)
        elif engine_task == "CliffWalking":
            iopt = 1 if kwargs.get("is_slippery", False) else 0
        elif engine_task == "Blackjack":
            iopt = (1 if kwargs.get("natural", False) else 0) | (2 if kwargs.get("sab", True) else 0)
        self.pool = _capi.CPool(engine_task, self.count, seed=seed,
                                max_episode_steps=kwargs.get("max_episode_steps", -1),
                                iopt=iopt, device=device, precision=precision,
                                env_id_offset=self.offset, **hc, **go)
        self.stream = torch.cuda.ExternalStream(self.pool.stream, device=f"cuda:{device}")
        self._full = None

    def reset_device(self):
        self.pool.reset_device()
        return self.pool.outputs_torch()

    def step_device(self, local_actions):
        """`local_actions`: this rank's [count, ...] slice of the global action batch."""
        self.pool.step_device(local_actions)
        return self.pool.outputs_torch()

    def all_gather(self, packed: bool = True):
        """The full batch of the last step on every rank (enqueued on the pool stream).
        packed=True: ONE all-gather of the packed slab, columns returned as
        `[world, n_local, ...]` views; packed=False: one all-gather per column into
        contiguous `[num_envs, ...]` tensors."""
        import torch

        from ._capi import _torch_view

        local = self.pool.outputs_torch()
        if self.world == 1:
            return local
        with torch.cuda.stream(self.stream):
            if not packed:
                self._full = all_gather_columns(local, self._full, self.group)
                return self._full
            slab = _torch_view(self.pool.outputs_device_ptr(), (self.pool.slab_bytes,),
                               torch.uint8, self.pool.device)
            self._full_slab = all_gather_packed(slab, getattr(self, "_full_slab", None),
                                                self.group)
        return packed_views(self._full_slab, self.pool.keys, self.count)

    # ------------------------------------------------------------------ peer exchange
    def enable_peer_exchange(self):
        """Allocate this rank's gather buffer and map every peer's (CUDA IPC handles travel
        through `all_gather_object`).  Collective: every rank must call it."""
        import torch.distributed as dist

        handle = self.pool.exchange_init(self.world, self.rank)
        if self.world > 1:
            handles = [None] * self.world
            dist.all_gather_object(handles, handle, group=self.group)
            self.pool.exchange_attach_ipc(handles)
            dist.barrier(group=self.group)
        self._peer = True

    def _gathered(self):
        import torch

        from ._capi import _torch_view

        ptr = self.pool.exchange_wait()
        full = _torch_view(ptr, (self.world, self.pool.exchange_slice_bytes), torch.uint8,
                           self.pool.device)
        return packed_views(full, self.pool.keys, self.count)

    def reset_exchange(self):
        """Forced reset of all local envs + exchange; views valid until the next call."""
        self.pool.step_exchange(None)
        return self._gathered()

    def step_exchange(self, local_actions):
        """Step the local envs and hand back the gathered batch of ALL ranks as
        `[world, n_local, ...]` views (enqueued on the pool stream, like step_device)."""
        self.pool.step_exchange(local_actions)
        return self._gathered()
