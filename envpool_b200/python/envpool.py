"""EnvPool mixin: mirror of envpool/python/envpool.py (send/recv/step/reset/async_reset)
plus the device-resident extension (step_device / reset_device / outputs) that hands the
consumer zero-copy torch views of the HBM output slab (SURVEY.md 8f.1)."""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Any, Dict, List, Optional

import numpy as np


def _normalize_env_id(env_id: Any) -> np.ndarray:
    if isinstance(env_id, np.ndarray):
        env_id = env_id.astype(np.int32, copy=False)
    elif hasattr(env_id, "astype"):
        env_id = env_id.astype(np.int32)
    else:
        env_id = np.asarray(env_id, dtype=np.int32)
    if getattr(env_id, "ndim", 0) == 0:
        env_id = env_id.reshape(1)
    return env_id


def _flatten_action_dict(action: Dict[str, Any], prefix: str = "") -> Dict[str, Any]:
    out: Dict[str, Any] = {}
    for k, v in action.items():
        key = f"{prefix}{k}"
        if isinstance(v, dict):
            out.update(_flatten_action_dict(v, key + "."))
        else:
            out[key] = v
    return out


class EnvPoolMixin(ABC):
    """Mixin class for EnvPool (envpool/python/envpool.py:59-384)."""

    _spec: Any

    def _player_action_count(self, adict: Dict[str, Any]) -> Optional[int]:
        """Rows of the player actions present in `adict` (envpool.py:82-101)."""
        count = None
        for key, spec in self.spec.action_array_spec.items():
            if key in ("env_id", "players.env_id") or key not in adict:
                continue
            shape = tuple(spec.shape)
            if len(shape) == 0 or shape[0] != -1:
                continue
            value_shape = np.shape(adict[key])
            rows = 1 if len(value_shape) == 0 else int(value_shape[0])
            if count is None:
                count = rows
            elif count != rows:
                raise RuntimeError("Inconsistent leading dimensions across player actions.")
        return count

    def _cached_players_env_id(self, env_id: np.ndarray,
                               player_count: int) -> Optional[np.ndarray]:
        """The player rows of `env_id` in the last recv, when they number `player_count`
        (envpool.py:103-121)."""
        if not hasattr(self, "_last_players_env_id"):
            return None
        cached = self._last_players_env_id
        segments = []
        for eid in env_id.tolist():
            matches = cached[cached == eid]
            if matches.size == 0:
                return None
            segments.append(matches)
        if not segments:
            return np.empty(0, dtype=np.int32)
        players_env_id = np.concatenate(segments)
        if players_env_id.shape[0] != player_count:
            return None
        return players_env_id

    def _infer_players_env_id(self, adict: Dict[str, Any]) -> np.ndarray:
        """players.env_id when the caller gives none (envpool.py:123-149): env_id itself for
        one action per env, else the last recv's player rows of those envs, else each env id
        repeated once per player."""
        env_id = _normalize_env_id(adict["env_id"])
        max_num_players = self.config.get("max_num_players", 1)
        if max_num_players == 1:
            return env_id
        player_count = self._player_action_count(adict)
        if player_count is None or player_count == env_id.shape[0]:
            return env_id
        cached = self._cached_players_env_id(env_id, player_count)
        if cached is not None:
            return cached
        if env_id.shape[0] == 0 or player_count % env_id.shape[0] != 0:
            raise RuntimeError("Cannot infer players.env_id for multiplayer action; "
                               "pass a dict action with explicit players.env_id.")
        players_per_env = player_count // env_id.shape[0]
        if players_per_env > max_num_players:
            raise RuntimeError("Cannot infer players.env_id for multiplayer action; "
                               "per-env player count exceeds max_num_players.")
        return np.repeat(env_id, players_per_env).astype(np.int32, copy=False)

    def _check_action(self, actions: List[np.ndarray]) -> None:
        if hasattr(self, "_check_action_finished"):  # only check once
            return
        self._check_action_finished = True
        for a, (k, v) in zip(actions, self.spec.action_array_spec.items()):
            if v.dtype != a.dtype:
                raise RuntimeError(f'Expected dtype {v.dtype} with action "{k}", got {a.dtype}')
            shape = tuple(v.shape)
            if len(shape) > 0 and shape[0] == -1:
                if a.shape[1:] != shape[1:]:
                    raise RuntimeError(
                        f'Expected shape {shape} with action "{k}", got {a.shape}')
            else:
                if len(a.shape) == 0 or a.shape[1:] != shape:
                    raise RuntimeError(
                        f'Expected shape {("num_env", *shape)} with action "{k}", got {a.shape}')

    def _from(self, action, env_id: Optional[np.ndarray] = None) -> List[np.ndarray]:
        """Convert action to the list the pybind `_send` takes (envpool.py:174-213)."""
        if isinstance(action, dict):
            adict = _flatten_action_dict(action)
        else:
            if not hasattr(self, "_last_action_type"):
                self._last_action_type = self._spec._action_spec[-1][0]
            if not hasattr(self, "_last_action_name"):
                self._last_action_name = self._spec._action_keys[-1]
            if isinstance(action, np.ndarray):
                # no copy when the caller already passes the spec dtype, C-contiguous
                action = action.astype(self._last_action_type, order="C", copy=False)
            adict = {self._last_action_name: action}
        if env_id is None:
            if "env_id" not in adict:
                adict["env_id"] = self.all_env_ids
        else:
            adict["env_id"] = _normalize_env_id(env_id)
        if "players.env_id" not in adict:
            adict["players.env_id"] = self._infer_players_env_id(adict)
        else:
            adict["players.env_id"] = _normalize_env_id(adict["players.env_id"])
        if not hasattr(self, "_action_names"):
            self._action_names = self._spec._action_keys
        return [adict[k] for k in self._action_names]

    def __len__(self) -> int:
        return self.config["num_envs"]

    @property
    def all_env_ids(self) -> np.ndarray:
        if not hasattr(self, "_all_env_ids"):
            self._all_env_ids = np.arange(self.config["num_envs"], dtype=np.int32)
        return self._all_env_ids

    @property
    def is_async(self) -> bool:
        return (self.config["batch_size"] > 0
                and self.config["num_envs"] != self.config["batch_size"])

    def seed(self, seed=None) -> None:
        warnings.warn("The `seed` function in envpool is abandoned. "
                      "You can set seed by envpool.make(..., seed=seed) instead.",
                      stacklevel=2)

    def render(self, env_ids=None, camera_id=None):
        raise RuntimeError("render is outside the accelerated step path of envpool_b200")

    def send(self, action, env_id: Optional[np.ndarray] = None) -> None:
        converted = self._from(action, env_id)
        self._check_action(converted)
        self._send(converted)

    def recv(self, reset: bool = False, return_info: bool = True):
        state_list = self._recv()
        if self.config.get("max_num_players", 1) > 1:
            # the player rows of this batch, for _infer_players_env_id (envpool.py:317-320)
            k = self._spec._state_keys.index("info:players.env_id")
            self._last_players_env_id = np.array(state_list[k], dtype=np.int32, copy=True)
        return self._to(state_list, reset, return_info)

    def async_reset(self) -> None:
        self._reset(self.all_env_ids)

    def step(self, action, env_id: Optional[np.ndarray] = None):
        self.send(action, env_id)
        return self.recv(reset=False, return_info=True)

    def reset(self, env_id: Optional[np.ndarray] = None):
        if env_id is None:
            env_id = self.all_env_ids
        self._reset(_normalize_env_id(env_id))
        return self.recv(reset=True, return_info=self.config["gym_reset_return_info"])

    def close(self) -> None:
        pass

    @property
    def config(self) -> Dict[str, Any]:
        return dict(zip(self._spec._config_keys, self._spec._config_values))

    def __repr__(self) -> str:
        import pprint

        config_str = ", ".join(f"{k}={pprint.pformat(v)}" for k, v in self.config.items())
        return f"{self.__class__.__name__}({config_str})"

    __str__ = __repr__

    # ------------------------------------------------------------------ device extension
    @property
    def device_pool(self):
        """Borrowed C-ABI view of this pool for the device-resident entry points."""
        if not hasattr(self, "_device_pool"):
            from .._capi import CPool

            self._device_pool = CPool.borrow(self._handle, self.config["num_envs"],
                                             device=self._device)
        return self._device_pool

    def step_device(self, action, env_id=None, stream=None):
        """One sync step with `action` (and optional `env_id`) already in HBM (torch CUDA
        tensors).  Returns {state_key: torch view} into the device output slab; the views
        are valid until the next step.  No host copy happens.

        `action` holds one row per env row, also in multi-player pools: there it is the action
        of the env's player to move (the first player row, as `send` resolves it).  A
        per-player column comes back as [n, players, ...]."""
        dp = self.device_pool
        dp.step_device(action, env_id, stream=stream)
        n = env_id.shape[0] if env_id is not None else None
        return dp.outputs_torch(n)

    def reset_device(self, env_id=None, stream=None):
        dp = self.device_pool
        dp.reset_device(env_id, stream=stream)
        n = env_id.shape[0] if env_id is not None else None
        return dp.outputs_torch(n)
