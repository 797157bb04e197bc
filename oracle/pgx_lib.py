"""TEST INFRASTRUCTURE ONLY: PGX TicTacToe-v1 / ConnectFour-v1 checkers, over two small native
libraries.

  libpgx_oracle.so     the C restatement of both games (pgx_oracle.c)            -> PgxOracle
  _ref/libpgx_ref.so   the reference's own AsyncEnvPool<TicTacToeEnv> /          -> PgxRef
                       <ConnectFourEnv>, two players, one worker thread,
                       compiled from an envpool checkout (ref_harness/pgx_driver.cc)

`build(reference_root)` compiles them (`__graft_entry__.build()` calls it); the oracle is also
built on first use.  The product package envpool_b200 never imports this module.

Both return the reference's 13 state columns as numpy arrays, per-player columns (leading -1 in
the spec) as [2 n, ...] player rows -- the players of env row i at rows 2 i and 2 i + 1 --
exactly as the reference's Recv and envpool_b200's `_recv` hand them out.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libpgx_oracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libpgx_ref.so")
_ORACLE_SRC = os.path.join(_HERE, "pgx_oracle.c")
_REF_SRC = os.path.join(_HERE, "ref_harness", "pgx_driver.cc")

GAMES = {"TicTacToe": 0, "ConnectFour": 1}
BOARD = {"TicTacToe": (3, 3), "ConnectFour": (6, 7)}
ACTIONS = {"TicTacToe": 9, "ConnectFour": 7}


def keys(game):
    """(name, dtype, row shape, per_player) of the state keys in the reference's order."""
    r, c = BOARD[game]
    return [
        ("info:env_id", np.int32, (), False), ("info:players.env_id", np.int32, (), True),
        ("elapsed_step", np.int32, (), False), ("done", np.bool_, (), False),
        ("reward", np.float32, (), True), ("discount", np.float32, (), True),
        ("step_type", np.int32, (), False), ("trunc", np.bool_, (), False),
        ("obs", np.bool_, (r, c, 2), True), ("info:board", np.int32, (r, c), False),
        ("info:current_player", np.int32, (), False),
        ("info:legal_action_mask", np.bool_, (ACTIONS[game],), False),
        ("info:players.id", np.int32, (), True),
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
                                                      "board_games.h")):
        os.makedirs(os.path.dirname(REF_SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-DNDEBUG", "-fPIC", "-shared",
                               "-pthread", "-I", os.path.join(_HERE, "ref_harness", "shims"),
                               "-I", reference_root, "-o", REF_SO, _REF_SRC])


_libs = {}


def _lib(path):
    if path not in _libs:
        if path != REF_SO:
            build()
        _libs[path] = ctypes.CDLL(path)
    return _libs[path]


def ref_available() -> bool:
    return os.path.exists(REF_SO)


def _collect(game, copy, n):
    out = {}
    for k, (name, dt, shape, per_player) in enumerate(keys(game)):
        arr = np.empty(((2 if per_player else 1) * n,) + shape, dtype=dt)
        copy(k, arr)
        out[name] = arr
    return out


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class PgxOracle:
    """CPU restatement of the engine's sync step of TicTacToe / ConnectFour: `step` takes one
    action per env row (the action of the env's first player row) and resets done envs."""

    def __init__(self, game, num_envs, seed=42, env_seed=None):
        L = _lib(ORACLE_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.pgo_create.restype = vp
        L.pgo_create.argtypes = [ci, ci, ci, vp]
        L.pgo_destroy.argtypes = [vp]
        L.pgo_reset.argtypes = [vp, vp, ci]
        L.pgo_step.argtypes = [vp, vp, vp, ci]
        L.pgo_column.restype = vp
        L.pgo_column.argtypes = [vp, ci]
        L.pgo_set_board.argtypes = [vp, ci, vp, ci, ci]
        self.L, self.game, self.n = L, game, num_envs
        self._env_seed = None if env_seed is None else _i32(env_seed)
        self.h = L.pgo_create(GAMES[game], num_envs, seed,
                              None if self._env_seed is None else self._env_seed.ctypes.data)
        if not self.h:
            raise RuntimeError("pgo_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.pgo_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self, n):
        def copy(k, arr):
            ctypes.memmove(arr.ctypes.data, self.L.pgo_column(self.h, k), arr.nbytes)
        return _collect(self.game, copy, n)

    def reset(self, env_ids=None):
        if env_ids is None:
            self.L.pgo_reset(self.h, None, self.n)
            return self._out(self.n)
        ids = _i32(env_ids)
        self.L.pgo_reset(self.h, ids.ctypes.data, len(ids))
        return self._out(len(ids))

    def step(self, action, env_ids=None):
        a = _i32(action)
        ids = None if env_ids is None else _i32(env_ids)
        n = self.n if ids is None else len(ids)
        assert a.size == n
        self.L.pgo_step(self.h, a.ctypes.data, None if ids is None else ids.ctypes.data, n)
        return self._out(n)

    def set_board(self, eid, board, color, current_player):
        """Put env `eid` in a crafted, running position (cells -1 / 0 / 1)."""
        b = _i32(board).ravel()
        self.L.pgo_set_board(self.h, eid, b.ctypes.data, color, current_player)


def first_player_actions(env_id, players_env_id, action):
    """The action row of each env row: the action of its first player row (the reference's
    ParseAction + `action["action"_][0]`)."""
    pid = np.asarray(players_env_id)
    out = np.empty(len(env_id), dtype=np.int32)
    for i, e in enumerate(np.asarray(env_id).tolist()):
        rows = np.flatnonzero(pid == e)
        if rows.size == 0:
            raise ValueError(f"env_id {e} has no row in players.env_id")
        out[i] = action[rows[0]]
    return out


class PgxRef:
    """The reference's own AsyncEnvPool<TicTacToeEnv> / <ConnectFourEnv> (needs
    _ref/libpgx_ref.so), two players, one worker thread unless num_threads says otherwise."""

    def __init__(self, game, num_envs, seed=42, num_threads=1):
        L = _lib(REF_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.pgr_create.restype = vp
        L.pgr_create.argtypes = [ci, ci, ci, ci]
        L.pgr_destroy.argtypes = [vp]
        L.pgr_reset.argtypes = [vp]
        L.pgr_step.argtypes = [vp, vp, ci, vp, vp, ci]
        L.pgr_num_keys.argtypes = [vp]
        L.pgr_key_bytes.restype = ctypes.c_uint64
        L.pgr_key_bytes.argtypes = [vp, ci]
        L.pgr_copy.argtypes = [vp, ci, vp]
        L.pgr_bench.restype = ctypes.c_double
        L.pgr_bench.argtypes = [vp, vp, ci, ci, ci]
        self.L, self.game, self.n = L, game, num_envs
        self.h = L.pgr_create(GAMES[game], num_envs, num_threads, seed)
        if not self.h:
            raise RuntimeError("pgr_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.pgr_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self):
        assert self.L.pgr_num_keys(self.h) == len(keys(self.game))

        def copy(k, arr):
            assert self.L.pgr_key_bytes(self.h, k) == arr.nbytes, keys(self.game)[k][0]
            self.L.pgr_copy(self.h, k, arr.ctypes.data)
        return _collect(self.game, copy, self.n)

    def reset(self):
        self.L.pgr_reset(self.h)
        return self._out()

    def step(self, action, env_id=None, players_env_id=None):
        """action: one per players.env_id row; env_id defaults to 0..n-1 and players.env_id to
        env_id.  Every env needs a player row."""
        ids = _i32(np.arange(self.n) if env_id is None else env_id)
        pids = ids if players_env_id is None else _i32(players_env_id)
        a = _i32(action)
        assert len(ids) == self.n and a.size == len(pids)
        missing = set(range(self.n)) - set(pids.tolist())
        if missing:
            raise ValueError(f"envs without a players.env_id row: {sorted(missing)[:4]}")
        self.L.pgr_step(self.h, ids.ctypes.data, len(ids), pids.ctypes.data, a.ctypes.data,
                        len(pids))
        return self._out()

    def bench(self, actions, warmup, steps):
        """actions: [T, N] stream; seconds for `steps` timed steps after `warmup`."""
        a = _i32(actions)
        return self.L.pgr_bench(self.h, a.ctypes.data, a.shape[0], warmup, steps)

    def hardware_concurrency(self):
        return self.L.pgr_hardware_concurrency()
