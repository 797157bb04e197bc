"""Key-tree helpers and space/spec stand-ins.

Mirrors envpool/python/data.py (to_nested_dict, to_namedtuple, dm_structure,
gym_structure, gym_spec_transform, dm_spec_transform).  The reference needs optree,
gymnasium and dm_env at import; none is installed in this image, so flatten/unflatten is
done with plain dict walks and, when gymnasium / dm_env are absent, minimal stand-in
classes with the same attributes are used.
"""
from __future__ import annotations

import keyword
import re
from collections import namedtuple
from typing import Any, Dict, List, NamedTuple, Tuple

import numpy as np

try:  # optional
    import gymnasium as _gymnasium
except Exception:  # pragma: no cover - not installed in this image
    _gymnasium = None
try:  # optional
    import dm_env as _dm_env
except Exception:  # pragma: no cover
    _dm_env = None

ACTION_THRESHOLD = 2**20


class ArraySpec:
    """Spec of one column (envpool/python/protocol.py:109-132)."""

    def __init__(self, dtype, shape, bounds, element_wise_bounds, is_discrete=False):
        self.dtype = np.dtype(dtype).type
        self.shape = list(shape)
        self.is_discrete = bool(is_discrete)
        if element_wise_bounds[0]:
            self.minimum = np.array(element_wise_bounds[0])
        else:
            self.minimum = bounds[0]
        if element_wise_bounds[1]:
            self.maximum = np.array(element_wise_bounds[1])
        else:
            self.maximum = bounds[1]

    def __repr__(self):
        return (f"ArraySpec(shape={self.shape}, dtype={self.dtype}, "
                f"minimum={self.minimum}, maximum={self.maximum})")


# ---- stand-ins used only when the real packages are missing --------------------------
class Box:
    def __init__(self, low, high, shape, dtype):
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self.low = np.broadcast_to(np.asarray(low, dtype=self.dtype), self.shape).copy()
        self.high = np.broadcast_to(np.asarray(high, dtype=self.dtype), self.shape).copy()

    # dm_env.specs.BoundedArray vocabulary (the same stand-in serves both adapters)
    @property
    def minimum(self):
        return self.low

    @property
    def maximum(self):
        return self.high

    def contains(self, x):
        x = np.asarray(x)
        return bool(x.shape == self.shape and np.all(x >= self.low) and np.all(x <= self.high))

    def __repr__(self):
        return f"Box({self.low.min()}, {self.high.max()}, {self.shape}, {self.dtype})"


class Discrete:
    def __init__(self, n, start=0):
        self.n = int(n)
        self.start = int(start)
        self.shape = ()
        self.dtype = np.dtype(np.int64)

    @property
    def num_values(self):  # dm_env.specs.DiscreteArray vocabulary
        return self.n

    def contains(self, x):
        return self.start <= int(x) < self.start + self.n

    def __repr__(self):
        return f"Discrete({self.n})" if self.start == 0 else f"Discrete({self.n}, start={self.start})"


class MultiBinary:
    """gymnasium.spaces.MultiBinary stand-in: the space of a bool column."""

    def __init__(self, n):
        self.n = n
        self.shape = tuple(int(s) for s in np.atleast_1d(n))
        self.dtype = np.dtype(np.int8)

    def contains(self, x):
        x = np.asarray(x)
        return bool(x.shape == self.shape and np.all((x == 0) | (x == 1)))

    def __repr__(self):
        return f"MultiBinary({self.n})"


class DictSpace(dict):
    """gymnasium.spaces.Dict stand-in: a dict of sub-spaces, also reachable as `.spaces`."""

    @property
    def spaces(self):
        return self

    def __repr__(self):
        return f"Dict({dict.__repr__(self)})"


def dict_space():
    """An empty gymnasium.spaces.Dict (or its stand-in), the container of a multi-key
    observation space (envpool/python/env_spec.py observation_space)."""
    return _gymnasium.spaces.Dict() if _gymnasium is not None else DictSpace()


class TimeStep(NamedTuple):
    """dm_env.TimeStep stand-in (same field order)."""
    step_type: Any
    reward: Any
    discount: Any
    observation: Any

    def first(self):
        return self.step_type == 0

    def mid(self):
        return self.step_type == 1

    def last(self):
        return self.step_type == 2


def make_timestep(step_type, reward, discount, observation):
    if _dm_env is not None:
        return _dm_env.TimeStep(step_type=step_type, reward=reward, discount=discount,
                                observation=observation)
    return TimeStep(step_type, reward, discount, observation)


# ---- envpool/python/data.py mirrors ----------------------------------------------------
def _maybe_scalar_int(value):
    arr = np.asarray(value)
    if arr.size != 1:
        return None
    scalar = arr.item()
    if not np.isfinite(scalar):
        return None
    integer = int(scalar)
    if not np.isclose(scalar, integer):
        return None
    return integer


def _maybe_discrete_range(spec: ArraySpec, spec_type: str):
    if np.prod(np.abs(spec.shape)) != 1:
        return None
    minimum = _maybe_scalar_int(spec.minimum)
    maximum = _maybe_scalar_int(spec.maximum)
    if minimum is None or maximum is None or maximum >= ACTION_THRESHOLD:
        return None
    if spec_type == "act":
        if not (spec.is_discrete or np.issubdtype(spec.dtype, np.integer)):
            return None
    elif not np.issubdtype(spec.dtype, np.integer):
        return None
    return minimum, maximum - minimum + 1


def to_nested_dict(flatten_dict: Dict[str, Any], generator: type = dict) -> Dict[str, Any]:
    ret = generator()
    for k, v in flatten_dict.items():
        segments = k.split(".")
        ptr = ret
        for s in segments[:-1]:
            keys = ptr.spaces if hasattr(ptr, "spaces") else ptr
            if s not in keys:
                ptr[s] = generator()
            ptr = ptr[s]
        ptr[segments[-1]] = v
    return ret


def _field(name: str) -> str:
    field = re.sub(r"\W", "_", name)
    if not field or field[0].isdigit() or keyword.iskeyword(field):
        field = f"_{field}"
    return field


def to_namedtuple(name: str, hdict: dict) -> tuple:
    field_names: List[str] = []
    used: Dict[str, int] = {}
    for key in hdict.keys():
        field = _field(key)
        if field in used:
            used[field] += 1
            field = f"{field}_{used[field]}"
        else:
            used[field] = 0
        field_names.append(field)
    return namedtuple(_field(name), field_names)(*[
        to_namedtuple(k, v) if isinstance(v, dict) else v for k, v in hdict.items()
    ])


def gym_spec_transform(name: str, spec: ArraySpec, spec_type: str):
    discrete_range = _maybe_discrete_range(spec, spec_type)
    shape = [s for s in spec.shape if s != -1]
    if _gymnasium is not None:
        if discrete_range is not None:
            return _gymnasium.spaces.Discrete(n=discrete_range[1], start=discrete_range[0])
        if np.issubdtype(spec.dtype, np.bool_):
            return _gymnasium.spaces.MultiBinary(shape)
        return _gymnasium.spaces.Box(shape=shape, dtype=spec.dtype, low=spec.minimum,
                                     high=spec.maximum)
    if discrete_range is not None:
        return Discrete(discrete_range[1], discrete_range[0])
    if np.issubdtype(spec.dtype, np.bool_):
        return MultiBinary(shape)
    return Box(spec.minimum, spec.maximum, shape, spec.dtype)


def dm_spec_transform(name: str, spec: ArraySpec, spec_type: str):
    discrete_range = _maybe_discrete_range(spec, spec_type)
    shape = [s for s in spec.shape if s != -1]
    if _dm_env is not None:
        if discrete_range is not None and discrete_range[0] == 0:
            return _dm_env.specs.DiscreteArray(
                name=name, num_values=discrete_range[1],
                dtype=spec.dtype if np.issubdtype(spec.dtype, np.integer) else np.int32)
        return _dm_env.specs.BoundedArray(name=name, shape=shape, dtype=spec.dtype,
                                          minimum=spec.minimum, maximum=spec.maximum)
    if discrete_range is not None and discrete_range[0] == 0:
        return Discrete(discrete_range[1], 0)
    return Box(spec.minimum, spec.maximum, shape, spec.dtype)


def gym_structure(keys: List[str]) -> Dict[str, Any]:
    """Nested dict whose leaves are the indices of `keys` (':' and '.' both nest)."""
    flat = {k.replace(":", "."): i for i, k in enumerate(keys)}
    return to_nested_dict(flat)


def dm_structure(root_name: str, keys: List[str]) -> Dict[str, Any]:
    """envpool/python/data.py:164-188: obs:* and info:* merge under `root_name`."""
    new_keys = []
    for key in keys:
        if key in ("obs", "info"):
            key = f"obs:{key}"
        key = key.replace("info:", "obs:")
        key = key.replace("obs:", f"{root_name}:")
        new_keys.append(key.replace(":", "."))
    return to_nested_dict({k: i for i, k in enumerate(new_keys)})


def fill_tree(tree: Dict[str, Any], values: List[Any]) -> Dict[str, Any]:
    """Replace index leaves by values (the optree.tree_unflatten of the reference)."""
    return {k: fill_tree(v, values) if isinstance(v, dict) else values[v]
            for k, v in tree.items()}
