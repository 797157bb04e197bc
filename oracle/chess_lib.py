"""TEST INFRASTRUCTURE ONLY: PGX Chess (Chess-v1) and GardnerChess (GardnerChess-v1) checkers,
beside go_lib's, over two small native libraries.

  libchess_oracle.so     the C restatement of ChessEnv / GardnerChessEnv (chess_oracle.c) -> ChessOracle
  _ref/libchess_ref.so   the reference's own AsyncEnvPool<ChessEnv> / <GardnerChessEnv>  -> ChessRef
                         through pgx_driver.cc's driver (ref_harness/chess_driver.cc), two
                         players, one worker thread, compiled from an envpool checkout

`build(reference_root)` compiles them (`__graft_entry__.build()` calls it); the oracle is also
built on first use.  The product package envpool_b200 never imports this module.

Both return the reference's state columns as numpy arrays, per-player columns as [2 n, ...] player
rows, exactly as pgx_lib's checkers do; `first_player_actions` is pgx_lib's.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from . import pgx_lib
from .pgx_lib import first_player_actions  # noqa: F401  (re-exported for the tests)

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libchess_oracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libchess_ref.so")
_ORACLE_SRC = os.path.join(_HERE, "chess_oracle.c")
_REF_SRC = os.path.join(_HERE, "ref_harness", "chess_driver.cc")

GAMES = {"Chess": 0, "GardnerChess": 1}  # task name -> game index of both libraries
SIZE = {"Chess": 8, "GardnerChess": 5}
PLANES = {"Chess": 73, "GardnerChess": 49}
CHANNELS = {"Chess": 119, "GardnerChess": 115}
MAX_STEPS = {"Chess": 512, "GardnerChess": 256}


def actions(game):
    return SIZE[game] ** 2 * PLANES[game]


def keys(game):
    """(name, dtype, row shape, per_player) of the state keys in the reference's order."""
    s = SIZE[game]
    common = [
        ("info:env_id", np.int32, (), False), ("info:players.env_id", np.int32, (), True),
        ("elapsed_step", np.int32, (), False), ("done", np.bool_, (), False),
        ("reward", np.float32, (), True), ("discount", np.float32, (), True),
        ("step_type", np.int32, (), False), ("trunc", np.bool_, (), False),
        ("obs", np.float32, (s, s, CHANNELS[game]), True), ("info:board", np.int32, (s, s), False),
    ]
    if game == "Chess":
        common.append(("info:castling_rights", np.bool_, (2, 2), False))
    common.append(("info:current_player", np.int32, (), False))
    if game == "Chess":
        common.append(("info:en_passant", np.int32, (), False))
    return common + [
        ("info:fullmove_count", np.int32, (), False), ("info:halfmove_count", np.int32, (), False),
        ("info:legal_action_mask", np.bool_, (actions(game),), False),
        ("info:players.id", np.int32, (), True), ("info:turn", np.int32, (), False),
    ]


def _stale(out, src):
    return not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out)


def build(reference_root: str = "") -> None:
    """Compile the oracle when stale and -- given an envpool checkout -- the reference driver
    into _ref/."""
    if _stale(ORACLE_SO, _ORACLE_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-o", ORACLE_SO,
                               _ORACLE_SRC])
    if reference_root and os.path.isfile(os.path.join(reference_root, "envpool", "pgx",
                                                      "chess_games.h")):
        os.makedirs(os.path.dirname(REF_SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-DNDEBUG", "-fPIC", "-shared",
                               "-pthread", "-I", os.path.join(_HERE, "ref_harness", "shims"),
                               "-I", os.path.join(_HERE, "ref_harness"), "-I", reference_root,
                               "-o", REF_SO, _REF_SRC])


_libs = {}


def _lib(path):
    if path not in _libs:
        if path != REF_SO:
            build()
        _libs[path] = ctypes.CDLL(path)
    return _libs[path]


def ref_available() -> bool:
    return os.path.exists(REF_SO)


def _collect(game, copy, n, with_obs=True):
    out = {}
    for k, (name, dt, shape, per_player) in enumerate(keys(game)):
        if name == "obs" and not with_obs:
            continue
        arr = np.empty(((2 if per_player else 1) * n,) + shape, dtype=dt)
        copy(k, arr)
        out[name] = arr
    return out


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class ChessOracle:
    """CPU restatement of the engine's sync step of Chess / GardnerChess: `step` takes one action
    per env row (the action of the env's first player row) and resets done envs.  With
    obs=False the obs column is neither computed nor returned."""

    def __init__(self, game, num_envs, seed=42, env_seed=None, obs=True):
        L = _lib(ORACLE_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.cho_create.restype = vp
        L.cho_create.argtypes = [ci, ci, ci, vp, ci]
        L.cho_destroy.argtypes = [vp]
        L.cho_reset.argtypes = [vp, vp, ci]
        L.cho_step.argtypes = [vp, vp, vp, ci]
        L.cho_column.restype = vp
        L.cho_column.argtypes = [vp, ci]
        L.cho_copy_env.argtypes = [vp, ci, ci]
        L.cho_label_target.argtypes = [vp, ci]
        L.cho_ended.argtypes = [vp, ci]
        L.cho_attacked.argtypes = [vp, ci, ci]
        self.L, self.game, self.n, self.with_obs = L, game, num_envs, obs
        self._env_seed = None if env_seed is None else _i32(env_seed)
        self.h = L.cho_create(GAMES[game], num_envs, seed,
                              None if self._env_seed is None else self._env_seed.ctypes.data,
                              1 if obs else 0)
        if not self.h:
            raise RuntimeError("cho_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.cho_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self, n):
        def copy(k, arr):
            ctypes.memmove(arr.ctypes.data, self.L.cho_column(self.h, k), arr.nbytes)
        return _collect(self.game, copy, n, self.with_obs)

    def reset(self, env_ids=None):
        if env_ids is None:
            self.L.cho_reset(self.h, None, self.n)
            return self._out(self.n)
        ids = _i32(env_ids)
        self.L.cho_reset(self.h, ids.ctypes.data, len(ids))
        return self._out(len(ids))

    def step(self, action, env_ids=None):
        a = _i32(action)
        ids = None if env_ids is None else _i32(env_ids)
        n = self.n if ids is None else len(ids)
        assert a.size == n
        self.L.cho_step(self.h, a.ctypes.data, None if ids is None else ids.ctypes.data, n)
        return self._out(n)

    def on_board(self):
        """bool[A]: the labels whose target lies on the board (the others move a piece off it)."""
        return np.array([self.L.cho_label_target(self.h, a) >= 0 for a in range(actions(self.game))])

    def ended(self, e):
        """Why env e's last in-range step ended its game: bit 0 no legal move, 1 in check, 2
        halfmove >= 100, 3 insufficient material, 4 threefold repetition, 5 the step limit."""
        return self.L.cho_ended(self.h, int(e))

    def attacked(self, e, sq):
        """Whether square sq of env e's board (the mover's frame) is attacked by the other side."""
        return bool(self.L.cho_attacked(self.h, int(e), int(sq)))

    def label_target(self, label):
        return self.L.cho_label_target(self.h, int(label))

    def copy_env(self, dst, src):
        """Env dst continues as a copy of env src's game (its RNG included)."""
        self.L.cho_copy_env(self.h, int(dst), int(src))


class ChessRef(pgx_lib.PgxRef):
    """The reference's own AsyncEnvPool<ChessEnv> / <GardnerChessEnv> (needs
    _ref/libchess_ref.so), two players, one worker thread unless num_threads says otherwise.
    Driven through pgx_lib.PgxRef's methods: the library carries pgx_driver.cc's entry points."""

    def __init__(self, game, num_envs, seed=42, num_threads=1):
        L = _lib(REF_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.pgr_create_chess.restype = vp
        L.pgr_create_chess.argtypes = [ci, ci, ci, ci]
        L.pgr_destroy.argtypes = [vp]
        L.pgr_reset.argtypes = [vp]
        L.pgr_step.argtypes = [vp, vp, ci, vp, vp, ci]
        L.pgr_num_keys.argtypes = [vp]
        L.pgr_key_bytes.restype = ctypes.c_uint64
        L.pgr_key_bytes.argtypes = [vp, ci]
        L.pgr_copy.argtypes = [vp, ci, vp]
        L.pgr_bench.restype = ctypes.c_double
        L.pgr_bench.argtypes = [vp, vp, ci, ci, ci]
        L.pgr_hardware_concurrency.restype = ci
        self.L, self.game, self.n = L, game, num_envs
        self.h = L.pgr_create_chess(GAMES[game], num_envs, num_threads, seed)
        if not self.h:
            raise RuntimeError("pgr_create_chess failed")

    def _out(self):
        assert self.L.pgr_num_keys(self.h) == len(keys(self.game))

        def copy(k, arr):
            assert self.L.pgr_key_bytes(self.h, k) == arr.nbytes, keys(self.game)[k][0]
            self.L.pgr_copy(self.h, k, arr.ctypes.data)
        return _collect(self.game, copy, self.n)
