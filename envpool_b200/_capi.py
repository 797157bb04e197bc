"""ctypes binding of the C ABI (include/envpool_b200.h) over envpool_b200/lib/libenvpool_b200.so.

This is the thinnest possible host: one Python method per C entry point.  The pybind11
modules (csrc/py_module.cc) bind the same symbols for the reference's `_XxxEnvPool`
classes; tests and bench.py use this module to reach the engine directly, including the
device-resident entry points (torch tensors supply device memory and streams only).

There is no CPU fallback: if the engine library is missing or no CUDA device is present,
loading or pool creation raises.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, List, Optional

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
ENGINE_SO = os.path.join(_PKG, "lib", "libenvpool_b200.so")

# enum epb_kind of the single-player kinds
KINDS = {
    "CartPole": 0, "Pendulum": 1, "Acrobot": 2, "MountainCar": 3,
    "MountainCarContinuous": 4, "FrozenLake": 5, "Catch": 6, "Taxi": 7,
    "NChain": 8, "CliffWalking": 9, "Blackjack": 10, "HalfCheetah": 11,
    "Game2048": 12, "Minesweeper": 13,
}
# ... and of the kinds with two players per env, whose per-player columns hold two rows per env
# row (epb_state_key_players).  Kept apart: code that walks KINDS sees one-player pools only.
TWO_PLAYER_KINDS = {"TicTacToe": 14, "ConnectFour": 15}
# ... and the two-player kinds added after those, with fixtures of their own
# (tests/golden/pgx/hex_othello/).
TWO_PLAYER_KINDS_2 = {"Hex": 16, "Othello": 17}
# every kind by task name but Go's
ALL_KINDS = {**KINDS, **TWO_PLAYER_KINDS, **TWO_PLAYER_KINDS_2}
# ... and Go, one kind per board size (tests/golden/pgx/go/); CPool takes its komi and
# max_terminal_steps
GO_KINDS = {"Go9x9": 18, "Go13x13": 19, "Go19x19": 20}
# ... and the chess games, Chess and GardnerChess (tests/test_pgx_chess.py)
CHESS_KINDS = {"Chess": 21, "GardnerChess": 22}
DTYPES = {0: np.int32, 1: np.float32, 2: np.float64, 3: np.bool_}

# every symbol include/envpool_b200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "epb_last_error", "epb_abi_version", "epb_create", "epb_destroy",
    "epb_num_state_keys", "epb_state_key", "epb_action_key", "epb_slab_bytes",
    "epb_num_envs", "epb_send", "epb_reset", "epb_recv_slab", "epb_recv_slab_ex", "epb_release_slab",
    "epb_recv", "epb_step_device", "epb_reset_device", "epb_outputs_device",
    "epb_rollout_device", "epb_step_many_device", "epb_sync", "epb_stream", "epb_state_bytes",
    "epb_state_layout", "epb_state_export", "epb_state_import", "epb_launch_count",
    "epb_bytes_per_env_step", "epb_exchange_init", "epb_exchange_base", "epb_exchange_attach",
    "epb_exchange_attach_ipc", "epb_step_exchange_device", "epb_exchange_wait",
    "epb_exchange_status", "epb_exchange_slice_bytes", "epb_exchange_depth",
    "epb_step_many_timed", "epb_step_exchange_many_device", "epb_fp64_peak_gflops",
    "epb_hc_model", "epb_hc_pair_rows", "epb_exchange_trace", "epb_game2048_boards",
    "epb_minesweeper_config", "epb_state_key_players", "epb_go_config",
]
IPC_HANDLE_BYTES = 64


class EpbConfig(ctypes.Structure):
    _fields_ = [
        ("num_envs", ctypes.c_int32), ("batch_size", ctypes.c_int32),
        ("seed", ctypes.c_int32), ("env_seed", ctypes.POINTER(ctypes.c_int32)),
        ("max_episode_steps", ctypes.c_int32), ("env_id_offset", ctypes.c_int32),
        ("device", ctypes.c_int32), ("precision", ctypes.c_int32),
        ("iopt", ctypes.c_int32), ("frame_skip", ctypes.c_int32),
        ("ctrl_cost_weight", ctypes.c_double),
        ("forward_reward_weight", ctypes.c_double),
        ("reset_noise_scale", ctypes.c_double),
    ]


class EpbKeyInfo(ctypes.Structure):
    _fields_ = [
        ("name", ctypes.c_char_p), ("dtype", ctypes.c_int32), ("ndim", ctypes.c_int32),
        ("shape", ctypes.c_int32 * 3), ("row_bytes", ctypes.c_int32),
        ("slab_offset", ctypes.c_int64),
    ]


_lib = None


def load_library() -> ctypes.CDLL:
    """dlopen the engine; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(ENGINE_SO):
        raise RuntimeError(
            f"{ENGINE_SO} is missing: build it with `python -m envpool_b200._build` "
            "(there is no CPU fallback for the env-step engine)")
    L = ctypes.CDLL(ENGINE_SO)
    vp, ci, pp = ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)
    L.epb_last_error.restype = ctypes.c_char_p
    L.epb_create.argtypes = [ci, ctypes.POINTER(EpbConfig), pp]
    L.epb_destroy.argtypes = [vp]
    L.epb_num_state_keys.argtypes = [vp]
    L.epb_state_key.argtypes = [vp, ci, ctypes.POINTER(EpbKeyInfo)]
    L.epb_state_key_players.argtypes = [vp, ci]
    L.epb_action_key.argtypes = [vp, ctypes.POINTER(EpbKeyInfo)]
    L.epb_slab_bytes.restype = ctypes.c_int64
    L.epb_slab_bytes.argtypes = [vp]
    L.epb_num_envs.argtypes = [vp]
    L.epb_send.argtypes = [vp, vp, vp, ci]
    L.epb_reset.argtypes = [vp, vp, ci]
    L.epb_recv_slab.argtypes = [vp, pp, ctypes.POINTER(ci)]
    L.epb_recv_slab_ex.argtypes = [vp, pp, ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.epb_release_slab.argtypes = [vp, vp]
    L.epb_recv.argtypes = [vp, pp, ctypes.POINTER(ci)]
    L.epb_step_device.argtypes = [vp, vp, vp, ci, vp]
    L.epb_reset_device.argtypes = [vp, vp, ci, vp]
    L.epb_outputs_device.argtypes = [vp, pp]
    L.epb_rollout_device.argtypes = [vp, vp, ci, pp, vp]
    L.epb_step_many_device.argtypes = [vp, vp, ci, ci, ci, ci, vp]
    L.epb_sync.argtypes = [vp]
    L.epb_stream.restype = vp
    L.epb_stream.argtypes = [vp]
    L.epb_state_bytes.restype = ctypes.c_int64
    L.epb_state_bytes.argtypes = [vp]
    L.epb_state_layout.argtypes = [vp, ctypes.POINTER(ctypes.c_int64)]
    L.epb_state_export.argtypes = [vp, vp]
    L.epb_state_import.argtypes = [vp, vp]
    L.epb_launch_count.restype = ctypes.c_int64
    L.epb_launch_count.argtypes = [vp]
    L.epb_bytes_per_env_step.argtypes = [vp]
    L.epb_exchange_init.argtypes = [vp, ci, ci, vp]
    L.epb_exchange_base.argtypes = [vp, pp, ctypes.POINTER(ctypes.c_int64)]
    L.epb_exchange_attach.argtypes = [vp, pp]
    L.epb_exchange_attach_ipc.argtypes = [vp, vp]
    L.epb_step_exchange_device.argtypes = [vp, vp, vp]
    L.epb_exchange_wait.argtypes = [vp, vp, pp]
    L.epb_exchange_status.argtypes = [vp, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ci)]
    L.epb_exchange_slice_bytes.restype = ctypes.c_int64
    L.epb_exchange_slice_bytes.argtypes = [vp]
    L.epb_exchange_depth.argtypes = [vp]
    L.epb_step_many_timed.argtypes = [vp, vp, ci, ci, ci, ci, ci, ci, ci, vp,
                                      ctypes.POINTER(ctypes.c_float)]
    L.epb_step_exchange_many_device.argtypes = [vp, vp, ci, ci, ci, ci, vp, pp]
    L.epb_fp64_peak_gflops.argtypes = [ci, ctypes.POINTER(ctypes.c_double)]
    L.epb_exchange_trace.argtypes = [vp, vp, ctypes.c_int64]
    L.epb_hc_model.restype = ctypes.c_int64
    L.epb_hc_model.argtypes = [vp, ctypes.c_int64]
    L.epb_hc_pair_rows.argtypes = [vp, ci]
    L.epb_game2048_boards.argtypes = [vp, vp, vp]
    L.epb_minesweeper_config.argtypes = [vp, vp, vp, vp, vp]
    L.epb_go_config.argtypes = [vp, ctypes.c_double, ctypes.c_int32]
    _lib = L
    return L


class EpbError(RuntimeError):
    pass


def hc_model_blob() -> bytes:
    """The compiled HalfCheetah model (hcm::HcModel) as bytes; host only, no GPU needed."""
    L = load_library()
    n = int(L.epb_hc_model(None, 0))
    buf = ctypes.create_string_buffer(n)
    L.epb_hc_model(buf, n)
    return buf.raw


def fp64_peak_gflops(device: int = 0) -> float:
    """Sustained fp64 FMA rate of the device (GFLOP/s), measured by the engine."""
    out = ctypes.c_double()
    _check(load_library().epb_fp64_peak_gflops(device, ctypes.byref(out)))
    return float(out.value)


def _check(rc: int):
    if rc != 0:
        msg = load_library().epb_last_error().decode()
        if rc == -1:
            raise ValueError(msg)
        raise EpbError(f"[{rc}] {msg}")


class Key:
    """One state or action column.  `shape` is the shape of an env row: a per-player column of a
    multi-player pool (`players` > 1) leads with the player dimension."""

    def __init__(self, info: EpbKeyInfo, players: int = 1):
        self.name = info.name.decode()
        self.dtype = np.dtype(DTYPES[info.dtype])
        self.players = players
        self.shape = tuple(info.shape[i] for i in range(info.ndim))
        if players > 1:
            self.shape = (players,) + self.shape
        self.row_bytes = info.row_bytes
        self.offset = info.slab_offset

    def __repr__(self):
        return f"Key({self.name}, {self.dtype}, {self.shape}, off={self.offset})"


class CPool:
    """One engine pool (one GPU's shard of envs) driven through the C ABI."""

    def __init__(self, task: str, num_envs: int, seed: int = 42,
                 max_episode_steps: int = -1, iopt: int = -1, device: int = 0,
                 precision: str = "f64", env_id_offset: int = 0,
                 env_seed=None, batch_size: int = 0, frame_skip: int = 0,
                 ctrl_cost_weight: float = math.nan, forward_reward_weight: float = math.nan,
                 reset_noise_scale: float = math.nan, komi: Optional[float] = None,
                 max_terminal_steps: Optional[int] = None):
        """HalfCheetah: frame_skip <= 0 and NaN weights / noise scale select the reference
        defaults (5, 0.1, 1.0, 0.1); every other value is used as given, negative included.
        Go: komi (default 7.5) and max_terminal_steps (default 0 = 2 S^2), epb_go_config."""
        L = load_library()
        self.lib = L
        cfg = EpbConfig()
        cfg.num_envs = num_envs
        cfg.batch_size = batch_size
        cfg.seed = seed
        self._env_seed = None
        if env_seed is not None and len(env_seed) > 0:
            self._env_seed = np.ascontiguousarray(env_seed, dtype=np.int32)
            if self._env_seed.shape[0] != num_envs:
                raise ValueError("`env_seed` must contain exactly one seed for each env")
            cfg.env_seed = self._env_seed.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        cfg.max_episode_steps = max_episode_steps
        cfg.env_id_offset = env_id_offset
        cfg.device = device
        cfg.precision = {"f64": 0, "f32": 1}[precision]
        cfg.iopt = iopt
        cfg.frame_skip = frame_skip
        cfg.ctrl_cost_weight = ctrl_cost_weight
        cfg.forward_reward_weight = forward_reward_weight
        cfg.reset_noise_scale = reset_noise_scale
        h = ctypes.c_void_p()
        kind = {**ALL_KINDS, **GO_KINDS, **CHESS_KINDS}[task]
        _check(L.epb_create(kind, ctypes.byref(cfg), ctypes.byref(h)))
        self.h = h
        self.task = task
        self.n = num_envs
        self.device = device
        self.precision = precision
        self._owned = True
        if komi is not None or max_terminal_steps is not None:
            self.go_config(7.5 if komi is None else komi,
                           0 if max_terminal_steps is None else max_terminal_steps)
        self._read_keys()

    @classmethod
    def borrow(cls, handle: int, num_envs: int, device: int = 0) -> "CPool":
        """Wrap an epb_pool* owned by someone else (a pybind _XxxEnvPool._handle)."""
        self = cls.__new__(cls)
        self.lib = load_library()
        self.h = ctypes.c_void_p(handle)
        self._owned = False
        self.n = num_envs
        self.device = device
        self._read_keys()
        return self

    def _read_keys(self):
        L, h = self.lib, self.h
        self.keys = []
        for k in range(L.epb_num_state_keys(h)):
            info = EpbKeyInfo()
            _check(L.epb_state_key(h, k, ctypes.byref(info)))
            self.keys.append(Key(info, L.epb_state_key_players(h, k)))
        info = EpbKeyInfo()
        _check(L.epb_action_key(h, ctypes.byref(info)))
        self.action_key = Key(info)
        self.slab_bytes = L.epb_slab_bytes(h)

    # ------------------------------------------------------------------ lifetime
    def close(self):
        if getattr(self, "h", None):
            if getattr(self, "_owned", True):
                self.lib.epb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ host path
    def send(self, action: np.ndarray, env_ids: Optional[np.ndarray] = None):
        a = np.ascontiguousarray(action, dtype=self.action_key.dtype)
        n = a.shape[0]
        ids = None
        if env_ids is not None:
            ids = np.ascontiguousarray(env_ids, dtype=np.int32)
            n = ids.shape[0]
        _check(self.lib.epb_send(self.h, a.ctypes.data,
                                 ids.ctypes.data if ids is not None else None, n))

    def reset_async(self, env_ids: Optional[np.ndarray] = None):
        if env_ids is None:
            _check(self.lib.epb_reset(self.h, None, self.n))
        else:
            ids = np.ascontiguousarray(env_ids, dtype=np.int32)
            _check(self.lib.epb_reset(self.h, ids.ctypes.data, ids.shape[0]))

    def recv(self) -> Dict[str, np.ndarray]:
        slab = ctypes.c_void_p()
        n, row0 = ctypes.c_int(), ctypes.c_int()
        _check(self.lib.epb_recv_slab_ex(self.h, ctypes.byref(slab), ctypes.byref(row0),
                                         ctypes.byref(n)))
        out = {}
        try:
            for k in self.keys:
                nbytes = k.row_bytes * n.value
                buf = (ctypes.c_char * nbytes).from_address(
                    slab.value + k.offset + row0.value * k.row_bytes)
                out[k.name] = np.frombuffer(buf, dtype=k.dtype).reshape(
                    (n.value,) + k.shape).copy()
        finally:
            _check(self.lib.epb_release_slab(self.h, slab))
        return out

    def reset(self, env_ids=None):
        self.reset_async(env_ids)
        return self.recv()

    def step(self, action, env_ids=None):
        self.send(action, env_ids)
        return self.recv()

    # ---------------------------------------------------------------- device path
    def _device_arg(self, t, what: str, dtype: np.dtype, rows: Optional[int], row_elems: int):
        """Device pointer of a caller-supplied buffer.  torch tensors are validated (a policy's
        argmax is int64, a sampled torque float64: reading those as int32/float32 rows would
        silently step on garbage) and converted when only dtype / layout differ; a raw integer
        pointer is taken on trust."""
        if not hasattr(t, "data_ptr"):
            return int(t), None, None
        import torch

        tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
               np.dtype(np.float64): torch.float64}[np.dtype(dtype)]
        if not t.is_cuda:
            raise ValueError(f"{what} must be a CUDA tensor (use step()/send() for host arrays)")
        if t.device.index != self.device:
            raise ValueError(f"{what} lives on cuda:{t.device.index}, the pool on "
                             f"cuda:{self.device}")
        if t.dtype != tdt:
            if t.dtype.is_floating_point != tdt.is_floating_point:
                raise ValueError(f"{what} has dtype {t.dtype}, the env expects {tdt}")
            t = t.to(tdt)
        if not t.is_contiguous():
            t = t.contiguous()
        have = t.shape[0] if t.dim() > 0 else 1
        if rows is not None and (t.numel() != rows * row_elems):
            raise ValueError(f"{what} has {t.numel()} elements, expected {rows} rows of "
                             f"{row_elems}")
        return t.data_ptr(), t, have

    def step_device(self, d_action, d_env_ids=None, n: Optional[int] = None, stream=None):
        """d_action / d_env_ids: torch CUDA tensors (validated; dtype / layout converted when
        needed) or raw device pointers (trusted).  env ids must lie in [0, num_envs)."""
        keep = []
        pi = None
        if d_env_ids is not None:
            pi, t, have = self._device_arg(d_env_ids, "env_id", np.int32, None, 1)
            keep.append(t)
            if n is None and have is not None:
                n = have
            if t is not None and n is not None and t.numel() < n:
                raise ValueError(f"env_id has {t.numel()} elements, n = {n}")
        if n is None:
            n = self.n
        row_elems = self.action_key.row_bytes // self.action_key.dtype.itemsize
        pa, t, _ = self._device_arg(d_action, "action", self.action_key.dtype, n, row_elems)
        keep.append(t)
        _check(self.lib.epb_step_device(self.h, pa, pi, n, stream))
        # converted temporaries must outlive the launch: park them until the next call
        self._keepalive = keep

    def reset_device(self, d_env_ids=None, n: Optional[int] = None, stream=None):
        pi, keep = None, None
        if d_env_ids is not None:
            pi, keep, have = self._device_arg(d_env_ids, "env_id", np.int32, None, 1)
            if n is None:
                n = have
        _check(self.lib.epb_reset_device(self.h, pi, n if n is not None else self.n, stream))
        self._keepalive = [keep]

    def outputs_device_ptr(self) -> int:
        p = ctypes.c_void_p()
        _check(self.lib.epb_outputs_device(self.h, ctypes.byref(p)))
        return p.value

    def outputs_torch(self, n: Optional[int] = None):
        """Zero-copy torch views of the device output slab (valid until the next step)."""
        import torch

        n = self.n if n is None else n
        base = self.outputs_device_ptr()
        out = {}
        tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
               np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
        for k in self.keys:
            out[k.name] = _torch_view(base + k.offset, (n,) + k.shape, tdt[k.dtype],
                                      self.device)
        return out

    def rollout_device(self, d_actions, T: int, d_cols, stream=None):
        """d_cols: list (len = num keys) of torch tensors / None, each [T, N, ...]."""
        arr = (ctypes.c_void_p * len(self.keys))()
        for i, c in enumerate(d_cols):
            arr[i] = c.data_ptr() if c is not None else None
        _check(self.lib.epb_rollout_device(self.h, d_actions.data_ptr(), T, arr, stream))

    def step_many_device(self, d_actions, t0: int, K: int, use_graph: bool = True,
                         stream=None):
        """K sync steps, actions cycled from the [T, N, ...] device stream `d_actions`."""
        _check(self.lib.epb_step_many_device(self.h, d_actions.data_ptr(),
                                             d_actions.shape[0], t0, K,
                                             1 if use_graph else 0, stream))

    def step_many_timed(self, d_actions, t0: int, K: int, mark0: int, mark1: int,
                        exchange: bool = False, use_graph: bool = True, stream=None) -> float:
        """The K-step chain with timestamps inside it: milliseconds for steps
        [mark0, mark1) in the chain's steady state (synchronises the stream)."""
        ms = ctypes.c_float()
        _check(self.lib.epb_step_many_timed(self.h, d_actions.data_ptr(), d_actions.shape[0],
                                            t0, K, mark0, mark1, 1 if exchange else 0,
                                            1 if use_graph else 0, stream, ctypes.byref(ms)))
        return float(ms.value)

    # ------------------------------------------------------------- peer exchange
    def exchange_init(self, world: int, rank: int) -> bytes:
        """Allocate this rank's gather buffer; returns its 64-byte CUDA IPC handle."""
        buf = ctypes.create_string_buffer(IPC_HANDLE_BYTES)
        _check(self.lib.epb_exchange_init(self.h, world, rank, buf))
        self.world, self.rank = world, rank
        return bytes(buf.raw)

    def exchange_base(self) -> int:
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        _check(self.lib.epb_exchange_base(self.h, ctypes.byref(p), ctypes.byref(n)))
        return p.value

    def exchange_attach(self, peer_bases: List[int]):
        """Same-process peers: raw base pointers of every rank's gather buffer."""
        arr = (ctypes.c_void_p * len(peer_bases))(*peer_bases)
        _check(self.lib.epb_exchange_attach(self.h, arr))

    def exchange_attach_ipc(self, handles: List[bytes]):
        """One process per GPU: the IPC handles of all ranks, rank order."""
        blob = b"".join(handles)
        if len(blob) != IPC_HANDLE_BYTES * len(handles):
            raise ValueError("every IPC handle must be 64 bytes")
        _check(self.lib.epb_exchange_attach_ipc(self.h, blob))

    def step_exchange(self, d_action, stream=None):
        """d_action None = forced reset of all envs."""
        pa = None if d_action is None else (
            d_action.data_ptr() if hasattr(d_action, "data_ptr") else int(d_action))
        _check(self.lib.epb_step_exchange_device(self.h, pa, stream))

    def exchange_wait(self, stream=None) -> int:
        """Enqueue the wait for all peers; returns the device pointer of [world][slab]."""
        p = ctypes.c_void_p()
        _check(self.lib.epb_exchange_wait(self.h, stream, ctypes.byref(p)))
        return p.value

    def step_exchange_many(self, d_actions, t0: int, K: int, use_graph: bool = True,
                           stream=None) -> int:
        """K exchanged steps (waits on a parallel graph branch); returns the device pointer
        of the last gathered batch, [world][exchange_slice_bytes]."""
        p = ctypes.c_void_p()
        _check(self.lib.epb_step_exchange_many_device(self.h, d_actions.data_ptr(),
                                                      d_actions.shape[0], t0, K,
                                                      1 if use_graph else 0, stream,
                                                      ctypes.byref(p)))
        return p.value

    @property
    def exchange_slice_bytes(self) -> int:
        return self.lib.epb_exchange_slice_bytes(self.h)

    @property
    def exchange_depth(self) -> int:
        return self.lib.epb_exchange_depth(self.h)

    def exchange_trace(self, steps: int) -> np.ndarray:
        """[steps, 8] device timestamps (ns) of the exchange kernels; needs
        ENVPOOL_B200_EXCHANGE_TRACE=1 at exchange_init (include/envpool_b200.h)."""
        out = np.zeros((steps, 8), dtype=np.int64)
        _check(self.lib.epb_exchange_trace(self.h, out.ctypes.data, steps))
        return out

    def exchange_status(self):
        steps, bad = ctypes.c_int64(), ctypes.c_int()
        _check(self.lib.epb_exchange_status(self.h, ctypes.byref(steps), ctypes.byref(bad)))
        return int(steps.value), bool(bad.value)

    def sync(self):
        _check(self.lib.epb_sync(self.h))

    @property
    def stream(self) -> int:
        return self.lib.epb_stream(self.h)

    @property
    def launch_count(self) -> int:
        return self.lib.epb_launch_count(self.h)

    @property
    def bytes_per_env_step(self) -> int:
        return self.lib.epb_bytes_per_env_step(self.h)

    def hc_pair_rows(self, n: Optional[int] = None) -> int:
        """HalfCheetah's two-lane kernel: constraint rows per lane held in shared memory for a
        launch of n batch rows (default num_envs); 0 for any other env or n outside
        [1, num_envs]."""
        return self.lib.epb_hc_pair_rows(self.h, self.n if n is None else n)

    def game2048_boards(self, initial=None, replay=None):
        """Game2048's configured boards, before the first reset: `initial` is 16 tile exponents
        (row-major), `replay` 32 boards of 16; None = not configured.  Cells outside [0, 26]
        raise ValueError."""
        ini = None if initial is None else np.ascontiguousarray(initial, dtype=np.int32).ravel()
        rep = None if replay is None else np.ascontiguousarray(replay, dtype=np.int32).ravel()
        if (ini is not None and ini.size != 16) or (rep is not None and rep.size != 512):
            raise ValueError("Game2048 boards: 16 initial cells and 32 x 16 replay cells")
        _check(self.lib.epb_game2048_boards(self.h, None if ini is None else ini.ctypes.data,
                                            None if rep is None else rep.ctypes.data))

    def minesweeper_config(self, mines=None, replay_boards=None, replay_rewards=None,
                           replay_done=None):
        """Minesweeper's configuration, before the first reset: `mines` 100 cells (nonzero =
        mine), `replay_boards` 32 boards of 100 cells, `replay_rewards` / `replay_done` 32 each
        (used only with replay boards); None = not configured.  Replay cells outside [-1, 8]
        raise ValueError."""
        bufs = []
        for v, dt, n in ((mines, np.int32, 100), (replay_boards, np.int32, 3200),
                         (replay_rewards, np.float32, 32), (replay_done, np.uint8, 32)):
            b = None if v is None else np.ascontiguousarray(v, dtype=dt).ravel()
            if b is not None and b.size != n:
                raise ValueError(f"Minesweeper config: expected {n} values, got {b.size}")
            bufs.append(b)
        _check(self.lib.epb_minesweeper_config(
            self.h, *[None if b is None else b.ctypes.data for b in bufs]))

    def go_config(self, komi: float, max_terminal_steps: int):
        """Go's komi and max_terminal_steps (0 = 2 S^2); before the pool's first reset, step,
        rollout or state import."""
        _check(self.lib.epb_go_config(self.h, float(komi), int(max_terminal_steps)))

    def state_layout(self) -> Dict[str, int]:
        out = (ctypes.c_int64 * 12)()
        _check(self.lib.epb_state_layout(self.h, out))
        names = ["flags", "mt_idx", "istate", "rstate", "mt", "NI", "NR", "real_size",
                 "rec", "rcons", "rprod", "rec_q"]
        return dict(zip(names, [int(v) for v in out]))

    def state_arrays(self, blob: np.ndarray) -> Dict[str, np.ndarray]:
        """Typed views into an exported state blob (writes go through to `blob`)."""
        lay, n = self.state_layout(), self.n
        real = np.float64 if lay["real_size"] == 8 else np.float32
        out = {"flags": blob[lay["flags"]:lay["flags"] + 4 * n].view(np.int32),
               "mt_idx": blob[lay["mt_idx"]:lay["mt_idx"] + 4 * n].view(np.int32),
               # chunked table: [78 chunks][n envs][8 words]
               "mt": blob[lay["mt"]:lay["mt"] + 4 * n * 624].view(np.uint32).reshape(78, n, 8)}
        if lay["NI"]:
            out["istate"] = blob[lay["istate"]:lay["istate"] + 4 * n * lay["NI"]].view(
                np.int32).reshape(lay["NI"], n)
        if lay["NR"]:
            nb = lay["real_size"] * n * lay["NR"]
            out["rstate"] = blob[lay["rstate"]:lay["rstate"] + nb].view(real).reshape(
                lay["NR"], n)
        if lay["rec"] >= 0:
            # reset-ahead record rings: rec[e, i % Q] = the env's i-th initial state,
            # records rcons[e] .. rprod[e] - 1 (uint8 counters, mod 256) are valid
            q = lay["rec_q"]
            nb = lay["real_size"] * n * lay["NR"] * q
            out["rec"] = blob[lay["rec"]:lay["rec"] + nb].view(real).reshape(n, q, lay["NR"])
            out["rcons"] = blob[lay["rcons"]:lay["rcons"] + n]
            out["rprod"] = blob[lay["rprod"]:lay["rprod"] + n]
        return out

    def state_export(self) -> np.ndarray:
        buf = np.empty(self.lib.epb_state_bytes(self.h), dtype=np.uint8)
        _check(self.lib.epb_state_export(self.h, buf.ctypes.data))
        return buf

    def state_import(self, blob: np.ndarray):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        if blob.nbytes != self.lib.epb_state_bytes(self.h):
            raise ValueError("state blob size mismatch")
        _check(self.lib.epb_state_import(self.h, blob.ctypes.data))


class _CudaArrayInterface:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {
            "data": (ptr, False), "shape": tuple(shape), "typestr": typestr,
            "version": 3, "strides": None,
        }


def _torch_view(ptr: int, shape, dtype, device: int):
    """Wrap raw device memory as a torch tensor without copying."""
    import torch

    typestr = {torch.int32: "<i4", torch.float32: "<f4", torch.float64: "<f8",
               torch.bool: "|b1", torch.uint8: "|u1"}[dtype]
    holder = _CudaArrayInterface(ptr, shape, typestr)
    return torch.as_tensor(holder, device=f"cuda:{device}")
