"""GPU: the peer exchange (include/envpool_b200.h "peer exchange", csrc/exchange.cuh) on ONE
device -- two pools play rank 0 and rank 1 of a 2-way env-id sharding, attached to each
other's gather buffers by raw pointer, each on its own stream.  After every step both
ranks must hold the oracle's full batch (integer envs bit-exact).  The multi-process /
CUDA-IPC flavour of the same path is tests/test_gpu_sharded.py (needs 2 GPUs)."""
import numpy as np
import pytest

from helpers import assert_batch_equal

pytestmark = pytest.mark.gpu


def _views(pool, ptr, world, n_local):
    import torch

    from envpool_b200._capi import _torch_view
    from envpool_b200.sharded import packed_views

    full = _torch_view(ptr, (world, pool.exchange_slice_bytes), torch.uint8, pool.device)
    return packed_views(full, pool.keys, n_local)


@pytest.mark.parametrize("task,kw,n_act", [
    ("FrozenLake", dict(max_episode_steps=100, iopt=4), 4),
    ("CartPole", dict(max_episode_steps=200), 2),
    ("Catch", dict(), 3),
])
def test_two_ranks_one_device(task, kw, n_act):
    import torch

    from envpool_b200._capi import CPool
    from oracle.oracle_lib import OraclePool

    n, world = 1000, 2          # not a multiple of the CTA size: exercises the padded tail
    pools = [CPool(task, n, seed=3, env_id_offset=r * n, **kw) for r in range(world)]
    orc = OraclePool(task, world * n, seed=3, **kw)
    for r, p in enumerate(pools):
        assert len(p.exchange_init(world, r)) == 64
    bases = [p.exchange_base() for p in pools]
    for p in pools:
        p.exchange_attach(bases)
    rng = np.random.default_rng(1)
    want = orc.reset()
    acts = None
    for t in range(40):
        d_acts = None if acts is None else [
            torch.from_numpy(acts[r * n:(r + 1) * n].copy()).cuda() for r in range(world)]
        torch.cuda.synchronize()
        for r, p in enumerate(pools):          # all pushes are enqueued before any wait
            p.step_exchange(None if d_acts is None else d_acts[r])
        ptrs = [p.exchange_wait() for p in pools]
        for p in pools:
            p.sync()
        for r, p in enumerate(pools):
            got = {k: v.reshape((world * n,) + tuple(v.shape[2:])).cpu().numpy()
                   for k, v in _views(p, ptrs[r], world, n).items()}
            assert_batch_equal(got, want, task, 1e-5 if task == "CartPole" else 0.0,
                               f"{task} rank {r} step {t}")
        acts = rng.integers(0, n_act, size=world * n).astype(np.int32)
        want = orc.step(acts)
    for p in pools:
        steps, timed_out = p.exchange_status()
        assert steps == 40 and not timed_out
        assert p.outputs_device_ptr() != 0
    for p in pools:
        p.close()


@pytest.mark.parametrize("task", ["CartPole", "Catch"], ids=lambda t: f"{t}-side")
def test_captured_exchange_chain_runs_ahead_of_the_waits(task):
    """epb_step_exchange_many_device: K exchanged steps in one CUDA graph, the waits on a
    parallel branch, so step t+1..t+depth-2 compute and push while the batch of step t is
    still arriving (ring slots + credit / ack flags).  After every chain both ranks hold the
    oracle's full batch; the un-captured chain gives the same bytes.  The captured chain issues
    the peer stores from a copy kernel on a side branch, so the step chain itself never waits
    for NVLink.

    Runs in a subprocess (tests/exchange_chain_check.py) with CUDA_DEVICE_MAX_CONNECTIONS=32:
    two ranks played by ONE process on ONE device share that process's hardware launch queues,
    and a wait kernel spinning at the head of a queue that also carries the other rank's step
    kernels is a false dependency the real deployment (one process per GPU) cannot have --
    there a rank only ever waits for kernels of other processes.  The cross-process flavour of
    the same chain is tests/test_gpu_sharded.py."""
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32",
               ENVPOOL_B200_EXCHANGE_TIMEOUT_S="20")
    out = subprocess.run([sys.executable, os.path.join(here, "exchange_chain_check.py"), task],
                         capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "CHAIN OK" in out.stdout, out.stdout[-3000:]


def test_exchange_errors_and_single_rank():
    import torch

    from envpool_b200._capi import CPool, EpbError

    p = CPool("NChain", 64, seed=0)
    with pytest.raises(EpbError):
        p.step_exchange(None)                  # not initialised
    with pytest.raises(ValueError):
        p.exchange_init(17, 0)                 # world out of range
    with pytest.raises(ValueError):
        p.exchange_init(2, 2)                  # rank out of range
    p.exchange_init(2, 0)
    with pytest.raises(EpbError):
        p.exchange_init(2, 0)                  # twice
    with pytest.raises(EpbError):
        p.step_exchange(None)                  # peers not attached
    p.close()

    # world == 1 degenerates to a plain step into the gather buffer
    q, ref = CPool("NChain", 64, seed=0), CPool("NChain", 64, seed=0)
    q.exchange_init(1, 0)
    with pytest.raises(EpbError):
        q.exchange_wait()                      # nothing exchanged yet
    a = torch.zeros(64, dtype=torch.int32, device="cuda")
    for t in range(5):
        q.step_exchange(None if t == 0 else a)
        ptr = q.exchange_wait()
        q.sync()
        ref.reset_device() if t == 0 else ref.step_device(a)
        ref.sync()
        got = _views(q, ptr, 1, 64)
        for k, v in ref.outputs_torch().items():
            assert torch.equal(got[k][0], v), k
    # flow control: at most depth - 1 exchanged steps may be outstanding
    for _ in range(q.exchange_depth - 1):
        q.step_exchange(a)
    with pytest.raises(EpbError):
        q.step_exchange(a)
    for _ in range(q.exchange_depth - 1):
        q.exchange_wait()
    with pytest.raises(EpbError):
        q.exchange_wait()
    q.sync()
    assert q.exchange_status() == (5 + q.exchange_depth - 1, False)
    q.close()
    ref.close()
