"""Jumanji family: binds the engine's pybind11 classes (`_Game2048EnvSpec` / `_Game2048EnvPool`,
`_MinesweeperEnvSpec` / `_MinesweeperEnvPool`, csrc/py_module.cc) to the Python adapters and
exports `XxxEnvSpec`, `XxxDMEnvPool` and `XxxGymnasiumEnvPool` for both -- the names
envpool/jumanji/__init__.py exports for those tasks."""
from ..python.api import py_env
from . import jumanji_envpool as _ext

Game2048EnvSpec, Game2048DMEnvPool, Game2048GymnasiumEnvPool = py_env(
    _ext._Game2048EnvSpec, _ext._Game2048EnvPool)
MinesweeperEnvSpec, MinesweeperDMEnvPool, MinesweeperGymnasiumEnvPool = py_env(
    _ext._MinesweeperEnvSpec, _ext._MinesweeperEnvPool)

__all__ = ["Game2048EnvSpec", "Game2048DMEnvPool", "Game2048GymnasiumEnvPool",
           "MinesweeperEnvSpec", "MinesweeperDMEnvPool", "MinesweeperGymnasiumEnvPool"]
