"""PGX family: binds the engine's pybind11 classes (`_TicTacToeEnvSpec` / `_TicTacToeEnvPool`,
`_ConnectFourEnvSpec`, `_HexEnvSpec`, `_OthelloEnvSpec`, `_GoEnvSpec`, `_ChessEnvSpec`,
`_GardnerChessEnvSpec` and their pools,
csrc/py_module.cc) to
the Python adapters and exports `XxxEnvSpec`, `XxxDMEnvPool` and `XxxGymnasiumEnvPool` for each
-- the names envpool/pgx/__init__.py exports for those games.  All are two-player pools: per-player columns
(obs, reward, discount, info:players.env_id, info:players.id) hold two rows per env."""
from ..python.api import py_env
from . import pgx_envpool as _ext

TicTacToeEnvSpec, TicTacToeDMEnvPool, TicTacToeGymnasiumEnvPool = py_env(
    _ext._TicTacToeEnvSpec, _ext._TicTacToeEnvPool)
ConnectFourEnvSpec, ConnectFourDMEnvPool, ConnectFourGymnasiumEnvPool = py_env(
    _ext._ConnectFourEnvSpec, _ext._ConnectFourEnvPool)
HexEnvSpec, HexDMEnvPool, HexGymnasiumEnvPool = py_env(_ext._HexEnvSpec, _ext._HexEnvPool)
OthelloEnvSpec, OthelloDMEnvPool, OthelloGymnasiumEnvPool = py_env(
    _ext._OthelloEnvSpec, _ext._OthelloEnvPool)
GoEnvSpec, GoDMEnvPool, GoGymnasiumEnvPool = py_env(_ext._GoEnvSpec, _ext._GoEnvPool)
ChessEnvSpec, ChessDMEnvPool, ChessGymnasiumEnvPool = py_env(_ext._ChessEnvSpec, _ext._ChessEnvPool)
GardnerChessEnvSpec, GardnerChessDMEnvPool, GardnerChessGymnasiumEnvPool = py_env(
    _ext._GardnerChessEnvSpec, _ext._GardnerChessEnvPool)

__all__ = ["TicTacToeEnvSpec", "TicTacToeDMEnvPool", "TicTacToeGymnasiumEnvPool",
           "ConnectFourEnvSpec", "ConnectFourDMEnvPool", "ConnectFourGymnasiumEnvPool",
           "HexEnvSpec", "HexDMEnvPool", "HexGymnasiumEnvPool",
           "OthelloEnvSpec", "OthelloDMEnvPool", "OthelloGymnasiumEnvPool",
           "GoEnvSpec", "GoDMEnvPool", "GoGymnasiumEnvPool",
           "ChessEnvSpec", "ChessDMEnvPool", "ChessGymnasiumEnvPool",
           "GardnerChessEnvSpec", "GardnerChessDMEnvPool", "GardnerChessGymnasiumEnvPool"]
