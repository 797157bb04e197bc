"""TEST INFRASTRUCTURE ONLY: Jumanji Minesweeper-v0 checkers, over three small native libraries.

  libms_oracle.so      the C restatement of the env (ms_oracle.c)                -> MinesweeperOracle
  libms_std_rng.so     libstdc++'s std::shuffle on a std::mt19937                -> StdShuffle
                       (ref_harness/ms_std_rng.cc)
  _ref/libms_ref.so    the reference's own AsyncEnvPool<MinesweeperEnv>,         -> MinesweeperRef
                       compiled from an envpool checkout (ref_harness/ms_driver.cc)

`build(reference_root)` compiles them (`__graft_entry__.build()` calls it); the first two are also
built on first use.  The product package envpool_b200 never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libms_oracle.so")
STD_RNG_SO = os.path.join(_HERE, "libms_std_rng.so")
REF_SO = os.path.join(_HERE, "_ref", "libms_ref.so")
_ORACLE_SRC = os.path.join(_HERE, "ms_oracle.c")
_STD_SRC = os.path.join(_HERE, "ref_harness", "ms_std_rng.cc")
_REF_SRC = os.path.join(_HERE, "ref_harness", "ms_driver.cc")

# state keys in the reference's order (common keys of core/env_spec.h, then MinesweeperEnvFns)
KEYS = [
    ("info:env_id", np.int32, ()), ("info:players.env_id", np.int32, ()),
    ("elapsed_step", np.int32, ()), ("done", np.bool_, ()), ("reward", np.float32, ()),
    ("discount", np.float32, ()), ("step_type", np.int32, ()), ("trunc", np.bool_, ()),
    ("obs:board", np.int32, (10, 10)), ("obs:action_mask", np.bool_, (10, 10)),
    ("obs:num_mines", np.int32, ()), ("obs:step_count", np.int32, ()),
]


def _stale(out, src):
    return not os.path.exists(out) or os.path.getmtime(src) > os.path.getmtime(out)


def build(reference_root: str = "") -> None:
    """Compile the oracle and the libstdc++ shim when stale, and -- given an envpool checkout --
    the reference driver into _ref/."""
    if _stale(ORACLE_SO, _ORACLE_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-o", ORACLE_SO,
                               _ORACLE_SRC])
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


def _ptr(a):
    return None if a is None else a.ctypes.data


class MinesweeperOracle:
    """CPU restatement of AsyncEnvPool<MinesweeperEnv> in sync mode; step/reset return the 12
    state columns as numpy arrays.  The configuration is the parsed one: `mines` 100 cells
    (nonzero = mine; None or no mine = random), `replay` 32 x 100 cells (None = no replay),
    `rewards` / `done` 32 each."""

    def __init__(self, num_envs, seed=42, max_episode_steps=90, env_seed=None, mines=None,
                 replay=None, rewards=None, done=None):
        L = _lib(ORACLE_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.mso_create.restype = vp
        L.mso_create.argtypes = [ci, ci, vp, ci]
        L.mso_destroy.argtypes = [vp]
        L.mso_config.argtypes = [vp, vp, vp, vp, vp]
        L.mso_reset.argtypes = [vp, vp, ci]
        L.mso_step.argtypes = [vp, vp, vp, ci]
        L.mso_column.restype = vp
        L.mso_column.argtypes = [vp, ci]
        L.mso_set_rng.argtypes = [vp, ci, vp, ci]
        L.mso_draw.restype = ctypes.c_uint32
        L.mso_draw.argtypes = [vp, ci]
        L.mso_shuffle.argtypes = [vp, ci, vp]
        L.mso_set_board.argtypes = [vp, ci, vp]
        self.L, self.n = L, num_envs
        es = None
        if env_seed is not None:
            self._env_seed = np.ascontiguousarray(env_seed, dtype=np.int32)
            es = self._env_seed.ctypes.data
        self.h = L.mso_create(num_envs, seed, es, max_episode_steps)
        if not self.h:
            raise RuntimeError("mso_create failed")
        self.config(mines, replay, rewards, done)

    def close(self):
        if getattr(self, "h", None):
            self.L.mso_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def config(self, mines=None, replay=None, rewards=None, done=None):
        bufs = [None if v is None else np.ascontiguousarray(v, dtype=dt).ravel()
                for v, dt in ((mines, np.int32), (replay, np.int32), (rewards, np.float32),
                              (done, np.uint8))]
        if self.L.mso_config(self.h, *[_ptr(b) for b in bufs]):
            raise ValueError("Minesweeper replay cells must lie in [-1, 8]")

    def _out(self, n):
        def copy(k, arr):
            ctypes.memmove(arr.ctypes.data, self.L.mso_column(self.h, k), arr.nbytes)
        return _collect(copy, n)

    def reset(self, env_ids=None):
        if env_ids is None:
            self.L.mso_reset(self.h, None, self.n)
            return self._out(self.n)
        ids = np.ascontiguousarray(env_ids, dtype=np.int32)
        self.L.mso_reset(self.h, ids.ctypes.data, len(ids))
        return self._out(len(ids))

    def step(self, action, env_ids=None):
        """action: [n, 2] (row, column)."""
        a = np.ascontiguousarray(action, dtype=np.int32)
        ids = None if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32)
        n = self.n if ids is None else len(ids)
        assert a.size == 2 * n
        self.L.mso_step(self.h, a.ctypes.data, _ptr(ids), n)
        return self._out(n)

    def set_rng(self, eid, mt624, idx):
        """Load an engine state (624 words + read position) into env `eid`'s mt19937."""
        w = np.ascontiguousarray(mt624, dtype=np.uint32)
        self.L.mso_set_rng(self.h, eid, w.ctypes.data, idx)

    def draw(self, eid):
        return self.L.mso_draw(self.h, eid)

    def shuffle(self, eid):
        out = np.empty(100, np.int32)
        self.L.mso_shuffle(self.h, eid, out.ctypes.data)
        return out

    def set_board(self, eid, board):
        b = np.ascontiguousarray(board, dtype=np.int32).ravel()
        self.L.mso_set_board(self.h, eid, b.ctypes.data)


class StdShuffle:
    """A real std::mt19937 and libstdc++'s std::shuffle of iota(100)."""

    def __init__(self):
        L = _lib(STD_RNG_SO)
        vp = ctypes.c_void_p
        L.mss_create.restype = vp
        L.mss_destroy.argtypes = [vp]
        L.mss_set.argtypes = [vp, vp, ctypes.c_int]
        L.mss_next.restype = ctypes.c_uint32
        L.mss_next.argtypes = [vp]
        L.mss_shuffle.argtypes = [vp, vp]
        self.L, self.h = L, L.mss_create()

    def __del__(self):
        if getattr(self, "h", None):
            self.L.mss_destroy(self.h)
            self.h = None

    def set(self, mt624, idx):
        w = np.ascontiguousarray(mt624, dtype=np.uint32)
        self.L.mss_set(self.h, w.ctypes.data, idx)

    def next(self):
        return self.L.mss_next(self.h)

    def shuffle(self):
        out = np.empty(100, np.int32)
        self.L.mss_shuffle(self.h, out.ctypes.data)
        return out


class MinesweeperRef:
    """The reference's own AsyncEnvPool<MinesweeperEnv> in sync mode (needs _ref/libms_ref.so);
    the four config strings as the reference takes them."""

    def __init__(self, num_envs, seed=42, max_episode_steps=90, mine_locations="",
                 replay_boards="", replay_rewards="", replay_done="", num_threads=0):
        L = _lib(REF_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.msr_create.restype = vp
        L.msr_create.argtypes = [ci] * 4 + [ctypes.c_char_p] * 4
        L.msr_destroy.argtypes = [vp]
        L.msr_reset.argtypes = [vp]
        L.msr_step.argtypes = [vp, vp]
        L.msr_num_keys.argtypes = [vp]
        L.msr_key_bytes.restype = ctypes.c_uint64
        L.msr_key_bytes.argtypes = [vp, ci]
        L.msr_copy.argtypes = [vp, ci, vp]
        L.msr_bench.restype = ctypes.c_double
        L.msr_bench.argtypes = [vp, vp, ci, ci, ci]
        self.L, self.n = L, num_envs
        self.h = L.msr_create(num_envs, num_threads, seed, max_episode_steps,
                              mine_locations.encode(), replay_boards.encode(),
                              replay_rewards.encode(), replay_done.encode())
        if not self.h:
            raise RuntimeError("msr_create failed")

    def close(self):
        if getattr(self, "h", None):
            self.L.msr_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _out(self):
        assert self.L.msr_num_keys(self.h) == len(KEYS)

        def copy(k, arr):
            assert self.L.msr_key_bytes(self.h, k) == arr.nbytes, KEYS[k][0]
            self.L.msr_copy(self.h, k, arr.ctypes.data)
        return _collect(copy, self.n)

    def reset(self):
        self.L.msr_reset(self.h)
        return self._out()

    def step(self, action):
        a = np.ascontiguousarray(action, dtype=np.int32).reshape(self.n, 2)
        self.L.msr_step(self.h, a.ctypes.data)
        return self._out()

    def bench(self, actions, warmup, steps):
        """actions: [T, N, 2] stream; seconds for `steps` timed steps after `warmup`."""
        a = np.ascontiguousarray(actions, dtype=np.int32)
        return self.L.msr_bench(self.h, a.ctypes.data, a.shape[0], warmup, steps)

    def hardware_concurrency(self):
        return self.L.msr_hardware_concurrency()
