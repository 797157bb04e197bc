"""TEST INFRASTRUCTURE ONLY: PGX Go (Go9x9-v1, Go13x13-v1, Go19x19-v1) checkers, beside pgx_lib's
and hex_othello_lib's, over two small native libraries.

  libgo_oracle.so      the C restatement of GoEnv (go_oracle.c)                     -> GoOracle
  _ref/libgo_ref.so    the reference's own AsyncEnvPool<GoEnv> through pgx_driver.cc's -> GoRef
                       driver (ref_harness/go_driver.cc), two players, one worker thread,
                       compiled from an envpool checkout

`build(reference_root)` compiles them (`__graft_entry__.build()` calls it); the oracle is also
built on first use.  The product package envpool_b200 never imports this module.

Both return the reference's 18 state columns as numpy arrays, per-player columns as [2 n, ...]
player rows, exactly as pgx_lib's checkers do; `first_player_actions` is pgx_lib's.  Both take
komi and max_terminal_steps (0 = 2 S^2), as the registered `GoNxN-v1` kwargs do.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from . import pgx_lib
from .pgx_lib import first_player_actions  # noqa: F401  (re-exported for the tests)

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libgo_oracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libgo_ref.so")
_ORACLE_SRC = os.path.join(_HERE, "go_oracle.c")
_REF_SRC = os.path.join(_HERE, "ref_harness", "go_driver.cc")

GAMES = {"Go9x9": 9, "Go13x13": 13, "Go19x19": 19}  # task name -> board size
KOMI = 7.5


def actions(game):
    return GAMES[game] ** 2 + 1


def keys(game):
    """(name, dtype, row shape, per_player) of the state keys in the reference's order."""
    s = GAMES[game]
    return [
        ("info:env_id", np.int32, (), False), ("info:players.env_id", np.int32, (), True),
        ("elapsed_step", np.int32, (), False), ("done", np.bool_, (), False),
        ("reward", np.float32, (), True), ("discount", np.float32, (), True),
        ("step_type", np.int32, (), False), ("trunc", np.bool_, (), False),
        ("obs", np.bool_, (s, s, 17), True), ("info:board", np.int32, (s, s), False),
        ("info:current_player", np.int32, (), False),
        ("info:legal_action_mask", np.bool_, (s * s + 1,), False),
        ("info:ko", np.int32, (), False), ("info:is_psk", np.bool_, (), False),
        ("info:consecutive_pass_count", np.int32, (), False),
        ("info:black_area", np.int32, (), False), ("info:white_area", np.int32, (), False),
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
    if reference_root and os.path.isfile(os.path.join(reference_root, "envpool", "pgx", "go.h")):
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


def _collect(game, copy, n):
    out = {}
    for k, (name, dt, shape, per_player) in enumerate(keys(game)):
        arr = np.empty(((2 if per_player else 1) * n,) + shape, dtype=dt)
        copy(k, arr)
        out[name] = arr
    return out


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class GoOracle:
    """CPU restatement of the engine's sync step of Go: `step` takes one action per env row (the
    action of the env's first player row) and resets done envs."""

    def __init__(self, game, num_envs, seed=42, env_seed=None, komi=KOMI, max_terminal_steps=0):
        L = _lib(ORACLE_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.goo_create.restype = vp
        L.goo_create.argtypes = [ci, ci, ci, vp, ctypes.c_double, ci]
        L.goo_destroy.argtypes = [vp]
        L.goo_reset.argtypes = [vp, vp, ci]
        L.goo_step.argtypes = [vp, vp, vp, ci]
        L.goo_column.restype = vp
        L.goo_column.argtypes = [vp, ci]
        self.L, self.game, self.n = L, game, num_envs
        self._env_seed = None if env_seed is None else _i32(env_seed)
        self.h = L.goo_create(GAMES[game], num_envs, seed,
                              None if self._env_seed is None else self._env_seed.ctypes.data,
                              komi, max_terminal_steps)
        if not self.h:
            raise RuntimeError("goo_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.goo_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self, n):
        def copy(k, arr):
            ctypes.memmove(arr.ctypes.data, self.L.goo_column(self.h, k), arr.nbytes)
        return _collect(self.game, copy, n)

    def reset(self, env_ids=None):
        if env_ids is None:
            self.L.goo_reset(self.h, None, self.n)
            return self._out(self.n)
        ids = _i32(env_ids)
        self.L.goo_reset(self.h, ids.ctypes.data, len(ids))
        return self._out(len(ids))

    def step(self, action, env_ids=None):
        a = _i32(action)
        ids = None if env_ids is None else _i32(env_ids)
        n = self.n if ids is None else len(ids)
        assert a.size == n
        self.L.goo_step(self.h, a.ctypes.data, None if ids is None else ids.ctypes.data, n)
        return self._out(n)


class GoRef(pgx_lib.PgxRef):
    """The reference's own AsyncEnvPool<GoEnv> (needs _ref/libgo_ref.so), two players, one worker
    thread unless num_threads says otherwise.  Driven through pgx_lib.PgxRef's methods: the
    library carries pgx_driver.cc's entry points."""

    def __init__(self, game, num_envs, seed=42, num_threads=1, komi=KOMI, max_terminal_steps=0):
        L = _lib(REF_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.pgr_create_go.restype = vp
        L.pgr_create_go.argtypes = [ci, ctypes.c_double, ci, ci, ci, ci]
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
        self.h = L.pgr_create_go(GAMES[game], komi, max_terminal_steps, num_envs, num_threads, seed)
        if not self.h:
            raise RuntimeError("pgr_create_go failed")

    def _out(self):
        assert self.L.pgr_num_keys(self.h) == len(keys(self.game))

        def copy(k, arr):
            assert self.L.pgr_key_bytes(self.h, k) == arr.nbytes, keys(self.game)[k][0]
            self.L.pgr_copy(self.h, k, arr.ctypes.data)
        return _collect(self.game, copy, self.n)
