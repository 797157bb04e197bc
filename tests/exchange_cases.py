"""The peer exchange checked against un-exchanged twins (shared by test_gpu_exchange_kinds.py and
its subprocess body exchange_matrix_check.py).

W pools play the W ranks of one env-id sharding on ONE device.  W twin pools are built with the
same arguments and no exchange, and are driven through the non-exchanged form of the same entry
point on the same action slice.  An exchange is a copy -- only the common columns are rebuilt on
the receiver, from the packed wire word -- so after every call each rank's gathered [W, n] batch
must equal the W twins' outputs byte for byte in every column, for every kind and precision.
The twins themselves are held to the oracle at the suite's usual bars (exact for the integer
envs, FLOAT_ATOL_F64 with row_tolerance for classic f64; f32 and HalfCheetah have no
free-running bar and rely on the byte check).

Two ways to play the ranks:
  * all ranks in one process, attached by raw pointer (`Ranks(..., rank=None)`): only for direct
    exchanged steps, where every rank's step has finished before any wait is enqueued, so no wait
    ever spins;
  * one process per rank, attached through CUDA IPC like the one-process-per-GPU deployment
    (`Ranks(..., rank=r)` inside a torch.distributed gloo group; every process builds all W
    twins and checks its own gathered batch).  Chains and timed chains overlap the ranks' steps,
    pushes and waits by design, and a wait kernel spins until its peer's push has published.
    CUDA promises no concurrency between kernels of one process -- graph branches and streams
    may share a hardware queue -- so a wait that spins ahead of the very push it waits for in
    such a queue only ends at its time bound.  Kernels of different processes are time-sliced
    on the device, so there every spinning wait lets the peer's push run."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from helpers import (HC_DEFAULT, INT_TASKS, assert_batch_equal, assert_hc_env_algebra,
                     random_actions)
from oracle.pgx_lib import ACTIONS as PGX_ACTIONS
from test_gpu_parity import FLOAT_ATOL_F64


class Kind:
    """One env kind as the exchange tests drive it: a task, its pool arguments (a small
    max_episode_steps, so that envs reset within a few dozen steps) and its oracle."""

    def __init__(self, name, task, **kw):
        self.name, self.task, self.kw = name, task, kw

    @property
    def jumanji(self):
        return self.task in ("Game2048", "Minesweeper")

    def pool(self, n, offset, seed, precision="f64"):
        from envpool_b200 import _capi

        if self.task == "Game2048":
            import test_gpu_game2048 as g

            return g.make_pool(_capi, g.meta_for("replay_cycle", n, seed), env_id_offset=offset,
                               precision=precision)
        if self.task == "Minesweeper":
            import test_gpu_minesweeper as m

            return m.make_pool(_capi, m.meta_for("replay", n, seed), env_id_offset=offset,
                               precision=precision)
        return _capi.CPool(self.task, n, seed=seed, env_id_offset=offset, precision=precision,
                           **self.kw)

    def actions(self, rng, shape):
        if self.task == "Game2048":
            import test_gpu_game2048 as g

            return g.actions(rng, shape)
        if self.task == "Minesweeper":
            import test_gpu_minesweeper as m

            return m.actions(rng, shape)
        return random_actions(self.task, rng, shape)

    def oracle(self, ids, seed, precision):
        """(oracle pool over the global env ids `ids`, float tolerance), or None where no
        free-running bar exists (f32, HalfCheetah)."""
        if self.task == "HalfCheetah" or (precision == "f32" and not self.jumanji):
            return None
        if self.task == "Game2048":
            import test_game2048
            import test_gpu_game2048 as g

            assert np.array_equal(ids, np.arange(len(ids))), "the Game2048 oracle is not sampled"
            return test_game2048.oracle_for(g.meta_for("replay_cycle", len(ids), seed)), 0.0
        if self.task == "Minesweeper":
            import test_gpu_minesweeper as m
            import test_minesweeper

            assert np.array_equal(ids, np.arange(len(ids))), "the Minesweeper oracle is not sampled"
            return test_minesweeper.oracle_for(m.meta_for("replay", len(ids), seed)), 0.0
        from oracle.oracle_lib import OraclePool

        tol = 0.0 if self.task in INT_TASKS else FLOAT_ATOL_F64
        return OraclePool(self.task, len(ids), seed=seed, env_seed=ids + seed, **self.kw), tol


KINDS = {k.name: k for k in [
    Kind("CartPole", "CartPole", max_episode_steps=9),
    Kind("Pendulum", "Pendulum", max_episode_steps=11, iopt=1),
    Kind("Acrobot", "Acrobot", max_episode_steps=13),
    Kind("MountainCar", "MountainCar", max_episode_steps=10),
    Kind("MountainCarContinuous", "MountainCarContinuous", max_episode_steps=12),
    Kind("FrozenLake4", "FrozenLake", max_episode_steps=10, iopt=4),
    Kind("FrozenLake8", "FrozenLake", max_episode_steps=10, iopt=8),
    Kind("Catch", "Catch"),
    Kind("Taxi", "Taxi", max_episode_steps=12),
    Kind("NChain", "NChain", max_episode_steps=9),
    Kind("CliffWalking", "CliffWalking", max_episode_steps=11, iopt=0),
    Kind("CliffWalkingSlippery", "CliffWalking", max_episode_steps=11, iopt=1),
    Kind("Blackjack", "Blackjack"),
    Kind("Game2048", "Game2048"),
    Kind("Minesweeper", "Minesweeper"),
    Kind("HalfCheetah", "HalfCheetah", max_episode_steps=8),
]}
CLASSIC = ["CartPole", "Pendulum", "Acrobot", "MountainCar", "MountainCarContinuous"]


class PgxKind(Kind):
    """A PGX game.  `oracle` returns None because the twins' comparison here reads a single-row
    info:players.env_id; test_gpu_pgx.py holds the twins to the oracle instead."""

    def actions(self, rng, shape):
        a = rng.integers(-1, PGX_ACTIONS[self.task] + 1, size=shape)
        return np.where(rng.random(shape) < 0.9,
                        rng.integers(0, PGX_ACTIONS[self.task], size=shape), a).astype(np.int32)

    def oracle(self, ids, seed, precision):
        return None


# (kind, precision) whose wire columns captured exchanged chains push through push_kernel:
# every kind above, the classic kinds in f32 as well, and the two-player PGX games.
PUSHED = ([(KINDS[k], "f64") for k in KINDS] + [(KINDS[k], "f32") for k in CLASSIC] +
          [(PgxKind(g, g), "f64") for g in ("TicTacToe", "ConnectFour")])
# bench.py's configurations (TASKS: registered limits and iopt, seed 0)
BENCH_KINDS = {
    "CartPole": Kind("CartPole", "CartPole", max_episode_steps=500),
    "Pendulum": Kind("Pendulum", "Pendulum", max_episode_steps=200, iopt=1),
    "Acrobot": Kind("Acrobot", "Acrobot", max_episode_steps=500),
    "FrozenLake": Kind("FrozenLake", "FrozenLake", max_episode_steps=100, iopt=4),
    "Catch": Kind("Catch", "Catch"),
    "HalfCheetah": Kind("HalfCheetah", "HalfCheetah", max_episode_steps=1000),
}


def sample_ids(total):
    """Every global env id of a small pool; of a large one the first and last 4096 and a
    strided sample, so the last rank's envs (the ones rank 0 receives) are covered."""
    if total <= 1 << 16:
        return np.arange(total, dtype=np.int32)
    return np.unique(np.concatenate([np.arange(4096), np.arange(total - 4096, total),
                                     np.arange(4096, total - 4096, 1021)])).astype(np.int32)


def spinning_ctas(n, world, sms):
    """Wait-kernel CTAs that may spin on a peer flag, summed over the ranks
    (exchange_wait_launch: per_peer CTAs for each of the world - 1 peer slices)."""
    cap = max(16, (2 * sms) // (world - 1 if world > 1 else 1))
    per_peer = min(max((n // 4 + 255) // 256, 1), cap)
    return world * (world - 1) * per_peer


def assert_spin_bound(n, world):
    """Overlapped chains put every rank's waits on the device together: their spinning CTAs
    must leave at least half the device's resident CTA slots (256-thread CTAs) free."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got, limit = spinning_ctas(n, world, sms), sms * 2048 // 256 // 2
    assert got <= limit, f"{world} ranks of {n} envs spin {got} wait CTAs > {limit}"


class Ranks:
    """W exchanged ranks and their W twins over one kind (see the module docstring).  rank=None:
    this process plays every rank; rank=r: only rank r, in a gloo group of W processes.  A context
    manager: on a clean exit every exchanged pool must report (steps, not timed out); every pool
    is closed either way."""

    def __init__(self, kind, n, world, seed=3, precision="f64", T=16, act_seed=1, rank=None):
        import torch

        self.kind, self.n, self.W, self.seed, self.precision = kind, n, world, seed, precision
        self.rank = rank
        self.local = list(range(world)) if rank is None else [rank]
        self.pools = {r: kind.pool(n, r * n, seed, precision) for r in self.local}
        self.twins = [kind.pool(n, r * n, seed, precision) for r in range(world)]
        rng = np.random.default_rng(act_seed)
        self.acts = kind.actions(rng, (T, world * n))
        self.T = T
        self.d_acts = [torch.from_numpy(np.ascontiguousarray(self.acts[:, r * n:(r + 1) * n]))
                       .cuda() for r in range(world)]
        self.ids = sample_ids(world * n)
        self.d_ids = torch.from_numpy(self.ids).long().cuda()
        orc = kind.oracle(self.ids, seed, precision) if rank in (None, 0) else None
        self.orc, self.tol = orc if orc else (None, None)
        self.want = None
        self.steps = 0       # exchanged steps, the initial forced reset included
        self.t = 0           # action rows consumed so far
        self.attached = False
        self.depth = 0

    # ------------------------------------------------------------------ setup / teardown
    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        try:
            if exc_type is None and self.attached:
                self._barrier()
                for r, p in self.pools.items():
                    assert p.exchange_status() == (self.steps, False), (r, p.exchange_status())
                self._barrier()   # no peer stores into an allocation that is being freed
        finally:
            for p in list(self.pools.values()) + self.twins:
                p.close()

    def _barrier(self):
        if self.rank is not None:
            import torch.distributed as dist

            dist.barrier()

    def attach(self):
        if self.rank is None:
            for r, p in self.pools.items():
                p.exchange_init(self.W, r)
            bases = [p.exchange_base() for p in self.pools.values()]
            for p in self.pools.values():
                p.exchange_attach(bases)
        else:
            import torch.distributed as dist

            p = self.pools[self.rank]
            handles = [None] * self.W
            dist.all_gather_object(handles, p.exchange_init(self.W, self.rank))
            p.exchange_attach_ipc(handles)
            self._barrier()
        first = self.pools[self.local[0]]
        self.depth = first.exchange_depth
        self.slice = first.exchange_slice_bytes
        self.attached = True
        return self

    # ------------------------------------------------------------------ the oracle
    def _oracle_reset(self):
        if self.orc is not None:
            self.want = self.orc.reset()

    def _oracle_rows(self, t0, K):
        if self.orc is not None:
            for k in range(K):
                self.want = self.orc.step(self.acts[(t0 + k) % self.T][self.ids])

    def _all(self):
        """(rank, pool) of every pool of this process: exchanged ranks, then twins."""
        return list(self.pools.items()) + list(enumerate(self.twins))

    # ------------------------------------------------------------------ plain (no exchange)
    def plain_reset(self):
        for _, p in self._all():
            p.reset_device()
        self._oracle_reset()

    def plain_chain(self, t0, K, use_graph=True):
        for r, p in self._all():
            p.step_many_device(self.d_acts[r], t0, K, use_graph=use_graph)
        self._oracle_rows(t0, K)

    def plain_timed(self, t0, K, lead, use_graph=True):
        n_chain = lead + K
        for r, p in self._all():
            p.step_many_timed(self.d_acts[r], t0, n_chain, lead, n_chain, False, use_graph)
        self._oracle_rows(t0, n_chain)

    # ------------------------------------------------------------------ exchanged entry points
    def direct(self, row=None, ctx=""):
        """One direct exchanged step (row None: a forced reset through the exchange).  Every
        rank's step has finished before any wait is enqueued, so no wait ever spins."""
        import torch

        self._barrier()
        torch.cuda.synchronize()
        hc_before = None
        if self.kind.task == "HalfCheetah" and row is not None:
            hc_before = np.concatenate([tw.state_arrays(tw.state_export())["rstate"][0]
                                        for tw in self.twins])
        for r, p in self.pools.items():
            p.step_exchange(None if row is None else self.d_acts[r][row])
        torch.cuda.synchronize()
        self._barrier()
        ptrs = {r: p.exchange_wait() for r, p in self.pools.items()}
        for r, tw in enumerate(self.twins):
            if row is None:
                tw.reset_device()
            else:
                tw.step_device(self.d_acts[r][row])
        torch.cuda.synchronize()
        self.steps += 1
        if row is None:
            self._oracle_reset()
        else:
            self._oracle_rows(row, 1)
        self.check(ptrs, ctx or f"direct step {self.steps}")
        if hc_before is not None:
            got = self.gathered(ptrs[self.local[0]])
            assert_hc_env_algebra(got, hc_before, self.acts[row], HC_DEFAULT,
                                  ctx=f"{ctx} direct step {self.steps}")

    def reset(self):
        self.direct(None, "forced reset")

    def steps_direct(self, count):
        for _ in range(count):
            self.direct(self.t % self.T)
            self.t += 1

    def chain(self, K, use_graph=True):
        """K exchanged steps through epb_step_exchange_many_device from action row t; the twins
        run step_many_device(K) on the same rows."""
        import torch

        assert_spin_bound(self.n, self.W)
        self._barrier()
        t0 = self.t % self.T
        phase = self.steps % self.depth
        ptrs = {r: p.step_exchange_many(self.d_acts[r], t0, K, use_graph=use_graph)
                for r, p in self.pools.items()}
        for r, tw in enumerate(self.twins):
            tw.step_many_device(self.d_acts[r], t0, K, use_graph=use_graph)
        torch.cuda.synchronize()
        self.steps += K
        self.t += K
        self._oracle_rows(t0, K)
        assert ptrs == {r: self.slot_ptr(p) for r, p in self.pools.items()}
        self.check(ptrs, f"chain K={K} t0={t0} phase {phase} graph={use_graph} "
                         f"-> {self.steps} steps")
        return (K, t0, phase)

    def timed(self, K, lead, t0=None, use_graph=True):
        """epb_step_many_timed(exchange=1), marks at lead and lead + K, as bench.py's Timer._one
        drives it (bench passes t0 = 0; by default the chain continues from action row t).
        epb_step_many_timed synchronises its stream on the host, so each rank this process
        plays is driven from a thread of its own."""
        import torch

        assert_spin_bound(self.n, self.W)
        self._barrier()
        t0 = self.t % self.T if t0 is None else t0
        n_chain = lead + K
        phase = self.steps % self.depth

        def one(r):
            return self.pools[r].step_many_timed(self.d_acts[r], t0, n_chain, lead, n_chain,
                                                 True, use_graph)

        with ThreadPoolExecutor(len(self.local)) as ex:
            ms = list(ex.map(one, self.local))
        assert all(m > 0 for m in ms), ms
        for r, tw in enumerate(self.twins):
            tw.step_many_timed(self.d_acts[r], t0, n_chain, lead, n_chain, False, use_graph)
        torch.cuda.synchronize()
        self.steps += n_chain
        self.t = t0 + n_chain
        self._oracle_rows(t0, n_chain)
        self.check({r: self.slot_ptr(p) for r, p in self.pools.items()},
                   f"timed chain lead {lead} + K {K} t0={t0} phase {phase} "
                   f"-> {self.steps} steps")
        return (n_chain, t0, phase)

    # ------------------------------------------------------------------ checks
    def slot_ptr(self, p):
        """The gathered slot of the last exchanged step: base + ((steps - 1) % D) * W * slice."""
        return p.exchange_base() + ((self.steps - 1) % self.depth) * self.W * self.slice

    def gathered(self, ptr):
        import torch

        from envpool_b200._capi import _torch_view
        from envpool_b200.sharded import packed_views

        full = _torch_view(ptr, (self.W, self.slice), torch.uint8, 0)
        return {k: v.reshape((self.W * self.n,) + tuple(v.shape[2:])).cpu().numpy()
                for k, v in packed_views(full, self.twins[0].keys, self.n).items()}

    def check(self, ptrs, ctx):
        """ptrs: {rank: its gathered slot} for the ranks this process plays."""
        import torch

        from envpool_b200._capi import _torch_view

        keys = self.twins[0].keys
        for r, p in self.pools.items():   # a wait past its time bound explains wrong bytes
            assert p.exchange_status() == (self.steps, False), (ctx, r, p.exchange_status())
        twin_bytes = [_torch_view(tw.outputs_device_ptr(), (tw.slab_bytes,), torch.uint8, 0)
                      for tw in self.twins]
        for r in self.pools:
            full = _torch_view(ptrs[r], (self.W, self.slice), torch.uint8, 0)
            for g in range(self.W):
                for k in keys:
                    lo, hi = k.offset, k.offset + k.row_bytes * self.n
                    a, b = full[g, lo:hi], twin_bytes[g][lo:hi]
                    if not torch.equal(a, b):
                        i = int((a != b).nonzero()[0]) // k.row_bytes
                        raise AssertionError(
                            f"{self.kind.name} W={self.W} n={self.n} {ctx}: rank {r} holds a "
                            f"wrong `{k.name}` of rank {g}'s env {i} (global {g * self.n + i})")
        if self.orc is not None:
            got = {}
            for k in keys:
                col = torch.cat([tw.outputs_torch()[k.name] for tw in self.twins])
                got[k.name] = col[self.d_ids].cpu().numpy()
            want = dict(self.want, **{"info:env_id": self.ids, "info:players.env_id": self.ids})
            assert_batch_equal(got, want, self.kind.task, self.tol,
                               f"{self.kind.name} twins vs oracle, {ctx}")


def set_env(**kv):
    """Set (value) or clear (None) ENVPOOL_B200_* variables read at exchange_init."""
    for k, v in kv.items():
        k = "ENVPOOL_B200_" + k
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
