"""EnvSpec mixin + metaclass: mirror of envpool/python/env_spec.py."""
from __future__ import annotations

import pprint
from abc import ABC, ABCMeta
from collections import namedtuple
from typing import Any, Dict

from .data import (ArraySpec, dict_space, dm_spec_transform, gym_spec_transform,
                   to_namedtuple, to_nested_dict)


def check_key_duplication(cls: str, keytype: str, keys) -> None:
    """envpool/python/utils.py:20-29"""
    ukeys, counts = {}, []
    for k in keys:
        ukeys[k] = ukeys.get(k, 0) + 1
    dup = [k for k, c in ukeys.items() if c > 1]
    if dup:
        raise SystemError(f"{cls} c++ code error. {keytype} keys {dup} are duplicated. "
                          f"Please report to the author of {cls}.")


class EnvSpecMixin(ABC):
    """Mixin class for EnvSpec (envpool/python/env_spec.py:33-206)."""

    gen_config: type

    @property
    def config(self):
        return self.gen_config(*self._config_values)

    @property
    def reward_threshold(self):
        try:
            return self.config.reward_threshold
        except AttributeError:
            return None

    @property
    def state_array_spec(self) -> Dict[str, Any]:
        return dict(zip(self._state_keys, [ArraySpec(*s) for s in self._state_spec]))

    @property
    def action_array_spec(self) -> Dict[str, Any]:
        return dict(zip(self._action_keys, [ArraySpec(*s) for s in self._action_spec]))

    def observation_spec(self):
        spec = self.state_array_spec
        spec = {
            k.replace("obs:", "").replace("info:", ""):
                dm_spec_transform(k.replace(":", ".").split(".")[-1], v, "obs")
            for k, v in spec.items() if k.startswith(("obs", "info"))
        }
        return to_namedtuple("State", to_nested_dict(spec))

    def action_spec(self):
        spec = self.action_array_spec
        if len(spec) == 3:
            spec.pop("env_id")
            spec.pop("players.env_id")
            return dm_spec_transform(list(spec.keys())[0], list(spec.values())[0], "act")
        spec = {k: dm_spec_transform(k.split(".")[-1], v, "act") for k, v in spec.items()}
        return to_namedtuple("Action", to_nested_dict(spec))

    @property
    def observation_space(self):
        spec = self.state_array_spec
        spec = {
            k.replace("obs:", "").replace(":", "."):
                gym_spec_transform(k.replace(":", ".").split(".")[-1], v, "obs")
            for k, v in spec.items() if k.startswith("obs")
        }
        if len(spec) == 1:
            return list(spec.values())[0]
        return to_nested_dict(spec, dict_space)

    @property
    def action_space(self):
        spec = self.action_array_spec
        if len(spec) == 3:
            spec.pop("env_id")
            spec.pop("players.env_id")
            return gym_spec_transform(list(spec.keys())[0], list(spec.values())[0], "act")
        spec = {k: gym_spec_transform(k.split(".")[-1], v, "act") for k, v in spec.items()}
        return to_nested_dict(spec)

    gymnasium_observation_space = observation_space
    gymnasium_action_space = action_space

    def __repr__(self) -> str:
        config_info = pprint.pformat(self.config)[6:]
        return f"{self.__class__.__name__}{config_info}"


class EnvSpecMeta(ABCMeta):
    """envpool/python/env_spec.py:208-222"""

    def __new__(cls, name, parents, attrs):
        base = parents[0]
        parents = (base, EnvSpecMixin)
        raw_config_keys = base._config_keys
        check_key_duplication(name, "config", raw_config_keys)
        config_keys = [s.replace(".", "_") for s in raw_config_keys]
        defaults = base._default_config_values
        attrs["gen_config"] = namedtuple("Config", config_keys, defaults=defaults)
        return super().__new__(cls, name, parents, attrs)
