"""TEST INFRASTRUCTURE ONLY: Jumanji Game2048-v1 checkers, over three small native libraries.

  libg2048_oracle.so     the C restatement of the env (g2048_oracle.c)          -> Game2048Oracle
  libg2048_std_rng.so    libstdc++'s bernoulli + the random-cell assignment     -> StdRng
                         (ref_harness/g2048_std_rng.cc)
  _ref/libg2048_ref.so   the reference's own AsyncEnvPool<Game2048Env>,        -> Game2048Ref
                         compiled from an envpool checkout (ref_harness/g2048_driver.cc)

`build(reference_root)` compiles them (`__graft_entry__.build()` calls it); the first two are also
built on first use.  The product package envpool_b200 never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libg2048_oracle.so")
STD_RNG_SO = os.path.join(_HERE, "libg2048_std_rng.so")
REF_SO = os.path.join(_HERE, "_ref", "libg2048_ref.so")
_ORACLE_SRC = os.path.join(_HERE, "g2048_oracle.c")
_STD_SRC = os.path.join(_HERE, "ref_harness", "g2048_std_rng.cc")
_REF_SRC = os.path.join(_HERE, "ref_harness", "g2048_driver.cc")

# state keys in the reference's order (common keys of core/env_spec.h, then Game2048EnvFns)
KEYS = [
    ("info:env_id", np.int32, ()), ("info:players.env_id", np.int32, ()),
    ("elapsed_step", np.int32, ()), ("done", np.bool_, ()), ("reward", np.float32, ()),
    ("discount", np.float32, ()), ("step_type", np.int32, ()), ("trunc", np.bool_, ()),
    ("obs:board", np.int32, (4, 4)), ("obs:action_mask", np.bool_, (4,)),
    ("info:highest_tile", np.int32, ()),
]


def _stale(out, src):
    return not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out)


def build(reference_root: str = "") -> None:
    """Compile the oracle and the libstdc++ shim when stale, and -- given an envpool checkout --
    the reference driver into _ref/."""
    if _stale(ORACLE_SO, _ORACLE_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared",
                               "-ffp-contract=off", "-o", ORACLE_SO, _ORACLE_SRC, "-lm"])
    if _stale(STD_RNG_SO, _STD_SRC):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-o", STD_RNG_SO,
                               _STD_SRC])
    if reference_root and os.path.isdir(os.path.join(reference_root, "envpool", "jumanji")):
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


def _collect(copy, n):
    out = {}
    for k, (name, dt, shape) in enumerate(KEYS):
        arr = np.empty((n,) + shape, dtype=dt)
        copy(k, arr)
        out[name] = arr
    return out


class Game2048Oracle:
    """CPU restatement of AsyncEnvPool<Game2048Env> in sync mode; step/reset return the 11 state
    columns as numpy arrays.  add_random_cell = game2048_add_random_cell."""

    def __init__(self, num_envs, seed=42, max_episode_steps=1000, add_random_cell=True,
                 env_seed=None, initial=None, replay=None):
        L = _lib(ORACLE_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.g2o_create.restype = vp
        L.g2o_create.argtypes = [ci, ci, vp, ci, ci]
        L.g2o_destroy.argtypes = [vp]
        L.g2o_boards.argtypes = [vp, vp, vp]
        L.g2o_reset.argtypes = [vp, vp, ci]
        L.g2o_step.argtypes = [vp, vp, vp, ci]
        L.g2o_column.restype = vp
        L.g2o_column.argtypes = [vp, ci]
        L.g2o_set_rng.argtypes = [vp, ci, vp, ci]
        L.g2o_draw.restype = ctypes.c_uint32
        L.g2o_draw.argtypes = [vp, ci]
        L.g2o_bernoulli.argtypes = [vp, ci, ctypes.c_double]
        L.g2o_random_cell.argtypes = [vp, ci, ci, vp, vp]
        self.L, self.n = L, num_envs
        es = None
        if env_seed is not None:
            self._env_seed = np.ascontiguousarray(env_seed, dtype=np.int32)
            es = self._env_seed.ctypes.data
        self.h = L.g2o_create(num_envs, seed, es, max_episode_steps, 1 if add_random_cell else 0)
        if not self.h:
            raise RuntimeError("g2o_create failed")
        if initial is not None or replay is not None:
            self.boards(initial, replay)

    def close(self):
        if getattr(self, "h", None):
            self.L.g2o_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def boards(self, initial=None, replay=None):
        """game2048_initial_board (16 exponents) / game2048_replay_boards (32 x 16); None = not
        configured.  Cells outside [0, 26] raise ValueError."""
        bufs = [None if b is None else np.ascontiguousarray(b, dtype=np.int32).ravel()
                for b in (initial, replay)]
        if self.L.g2o_boards(self.h, *[None if b is None else b.ctypes.data for b in bufs]):
            raise ValueError("Game2048 boards: cells must lie in [0, 26]")

    def _out(self, n):
        def copy(k, arr):
            ctypes.memmove(arr.ctypes.data, self.L.g2o_column(self.h, k), arr.nbytes)
        return _collect(copy, n)

    def reset(self, env_ids=None):
        if env_ids is None:
            self.L.g2o_reset(self.h, None, self.n)
            return self._out(self.n)
        ids = np.ascontiguousarray(env_ids, dtype=np.int32)
        self.L.g2o_reset(self.h, ids.ctypes.data, len(ids))
        return self._out(len(ids))

    def step(self, action, env_ids=None):
        a = np.ascontiguousarray(action, dtype=np.int32)
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32)
        n = self.n if ids is None else len(ids)
        self.L.g2o_step(self.h, a.ctypes.data, None if ids is None else ids.ctypes.data, n)
        return self._out(n)

    def set_rng(self, eid, mt624, idx):
        """Load an engine state (624 words + read position) into env `eid`'s mt19937."""
        w = np.ascontiguousarray(mt624, dtype=np.uint32)
        self.L.g2o_set_rng(self.h, eid, w.ctypes.data, idx)

    def draw(self, eid):
        return self.L.g2o_draw(self.h, eid)

    def bernoulli(self, eid, prob):
        return bool(self.L.g2o_bernoulli(self.h, eid, prob))

    def random_cell(self, eid, n_empty):
        """AddRandomCell's draws for n_empty empty cells: (value, position)."""
        v, p = ctypes.c_int(), ctypes.c_int()
        self.L.g2o_random_cell(self.h, eid, n_empty, ctypes.byref(v), ctypes.byref(p))
        return v.value, p.value


class StdRng:
    """A real std::mt19937 with libstdc++'s bernoulli and the random-cell assignment."""

    def __init__(self):
        L = _lib(STD_RNG_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.g2s_create.restype = vp
        L.g2s_destroy.argtypes = [vp]
        L.g2s_set.argtypes = [vp, vp, ci]
        L.g2s_next.restype = ctypes.c_uint32
        L.g2s_next.argtypes = [vp]
        L.g2s_bernoulli.argtypes = [vp, ctypes.c_double]
        L.g2s_random_cell.argtypes = [vp, ci, vp, vp]
        self.L, self.h = L, L.g2s_create()

    def __del__(self):
        if getattr(self, "h", None):
            self.L.g2s_destroy(self.h)
            self.h = None

    def set(self, mt624, idx):
        w = np.ascontiguousarray(mt624, dtype=np.uint32)
        self.L.g2s_set(self.h, w.ctypes.data, idx)

    def next(self):
        return self.L.g2s_next(self.h)

    def bernoulli(self, prob):
        return bool(self.L.g2s_bernoulli(self.h, prob))

    def random_cell(self, n_empty):
        v, p = ctypes.c_int(), ctypes.c_int()
        self.L.g2s_random_cell(self.h, n_empty, ctypes.byref(v), ctypes.byref(p))
        return v.value, p.value


class Game2048Ref:
    """The reference's own AsyncEnvPool<Game2048Env> in sync mode (needs _ref/libg2048_ref.so)."""

    def __init__(self, num_envs, seed=42, max_episode_steps=1000, add_random_cell=True,
                 initial_board="", replay_boards="", num_threads=0):
        L = _lib(REF_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.g2r_create.restype = vp
        L.g2r_create.argtypes = [ci] * 5 + [ctypes.c_char_p] * 2
        L.g2r_destroy.argtypes = [vp]
        L.g2r_reset.argtypes = [vp]
        L.g2r_step.argtypes = [vp, vp]
        L.g2r_num_keys.argtypes = [vp]
        L.g2r_key_bytes.restype = ctypes.c_uint64
        L.g2r_key_bytes.argtypes = [vp, ci]
        L.g2r_copy.argtypes = [vp, ci, vp]
        L.g2r_bench.restype = ctypes.c_double
        L.g2r_bench.argtypes = [vp, vp, ci, ci, ci]
        self.L, self.n = L, num_envs
        self.h = L.g2r_create(num_envs, num_threads, seed, max_episode_steps,
                              1 if add_random_cell else 0, initial_board.encode(),
                              replay_boards.encode())
        if not self.h:
            raise RuntimeError("g2r_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.g2r_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self):
        assert self.L.g2r_num_keys(self.h) == len(KEYS)

        def copy(k, arr):
            assert self.L.g2r_key_bytes(self.h, k) == arr.nbytes, KEYS[k][0]
            self.L.g2r_copy(self.h, k, arr.ctypes.data)
        return _collect(copy, self.n)

    def reset(self):
        self.L.g2r_reset(self.h)
        return self._out()

    def step(self, action):
        a = np.ascontiguousarray(action, dtype=np.int32).reshape(self.n)
        self.L.g2r_step(self.h, a.ctypes.data)
        return self._out()

    def bench(self, actions, warmup, steps):
        """actions: [T, N] stream; seconds for `steps` timed steps after `warmup`."""
        a = np.ascontiguousarray(actions, dtype=np.int32)
        return self.L.g2r_bench(self.h, a.ctypes.data, a.shape[0], warmup, steps)

    def hardware_concurrency(self):
        return self.L.g2r_hardware_concurrency()
