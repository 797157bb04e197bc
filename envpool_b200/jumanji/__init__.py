"""Jumanji family: binds the engine's pybind11 classes (`_Game2048EnvSpec` / `_Game2048EnvPool`,
csrc/py_module.cc) to the Python adapters and exports `Game2048EnvSpec`, `Game2048DMEnvPool`
and `Game2048GymnasiumEnvPool` -- the names envpool/jumanji/__init__.py exports for Game2048."""
from ..python.api import py_env
from . import jumanji_envpool as _ext

Game2048EnvSpec, Game2048DMEnvPool, Game2048GymnasiumEnvPool = py_env(
    _ext._Game2048EnvSpec, _ext._Game2048EnvPool)

__all__ = ["Game2048EnvSpec", "Game2048DMEnvPool", "Game2048GymnasiumEnvPool"]
