"""CPU, world_size 2, gloo: the host-side logic of the multi-GPU path -- env-id block
partition, per-rank seeding by global id, and the all-gather that reassembles the full
batch in env-id order.  The per-shard "engine" here is the CPU oracle (no GPU in this
container); the same ShardedPool code path runs the CUDA engine under NCCL on the box
(bench.py --gpus N, tests/test_gpu_parity.py::test_full_size_properties for the math)."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shard_range():
    from envpool_b200.sharded import shard_range

    assert shard_range(1 << 20, 0, 8) == (0, 131072)
    assert shard_range(1 << 20, 7, 8) == (917504, 131072)
    assert [shard_range(32, r, 4) for r in range(4)] == [(0, 8), (8, 8), (16, 8), (24, 8)]
    with pytest.raises(ValueError):
        shard_range(10, 0, 3)
    with pytest.raises(ValueError):
        shard_range(8, 2, 2)


def _worker(rank, world, port, task, n_total, steps, ret):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    from envpool_b200.sharded import all_gather_columns, shard_range
    from oracle.oracle_lib import OraclePool

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=world)
    off, cnt = shard_range(n_total, rank, world)
    seed = 11
    # a shard is seeded by GLOBAL env id: seed + offset + local id
    shard = OraclePool(task, cnt, env_seed=[seed + off + e for e in range(cnt)],
                       max_episode_steps=100, iopt=4)
    full_ref = OraclePool(task, n_total, seed=seed, max_episode_steps=100, iopt=4)
    rng = np.random.default_rng(0)            # same stream on every rank
    ok = True
    loc, ref = shard.reset(), full_ref.reset()
    for t in range(steps + 1):
        loc["info:env_id"] = loc["info:env_id"] + off          # engine's env_id_offset
        loc["info:players.env_id"] = loc["info:players.env_id"] + off
        full = all_gather_columns({k: torch.from_numpy(v) for k, v in loc.items()})
        for k in ref:
            ok &= bool(np.array_equal(full[k].numpy(), ref[k]))
        a = rng.integers(0, 4, size=n_total).astype(np.int32)
        loc, ref = shard.step(a[off:off + cnt]), full_ref.step(a)
    ret[rank] = ok
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_all_gather_reassembles_full_batch():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, "FrozenLake", 64, 30, ret))
             for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert ret[0] is True and ret[1] is True


def test_sharded_pool_refuses_kwargs_it_cannot_carry(engine_built):
    """A task kwarg a shard's pool cannot take is refused, not dropped (the shard would run the
    default while the caller believes otherwise); so is HalfCheetah's frame_skip < 1, as make()
    refuses it.  All of it is decided before a device is touched."""
    from envpool_b200.sharded import ShardedPool

    for task, kw in (("Game2048-v1", dict(game2048_add_random_cell=False)),
                     ("Minesweeper-v0", dict(minesweeper_mine_locations="0,1,2")),
                     ("HalfCheetah-v4", dict(frame_stack=2)),
                     ("HalfCheetah-v4", dict(exclude_current_positions_from_observation=False)),
                     ("CartPole-v1", dict(frame_skip=2)),
                     ("HalfCheetah-v4", dict(frame_skip=0)),
                     ("HalfCheetah-v5", dict(frame_skip=-1))):
        with pytest.raises(ValueError):
            ShardedPool(task, 64, **kw)
