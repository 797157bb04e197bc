"""GPU: chained steps store only the common columns that change (csrc/common.cuh write_common,
step_kernel's prev_in_slab, set by capi.cu run_chain for the steps after a chain's first).
Each chain starts from an output slab filled with 0xFF, so a column that a chain's first step
failed to store, or that a later step left stale, shows up.  After chains of K = 1, 2, 9 and
40 steps, captured (and then replayed) and uncaptured, every output column equals the same
steps launched one by one with step_device, which stores every column.  The pools' short
max_episode_steps make envs truncate, reset and restart inside the chains; CartPole3
(max_episode_steps = 3) flips step_type 0 -> 1 -> 2, discount and trunc every few steps.

The CTA size of the step kernel is read once per process (ENVPOOL_B200_STEP_BLOCK), so each
size runs in a subprocess of its own: `python tests/test_gpu_chain_stores.py chains`."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
from exchange_cases import KINDS, Kind  # noqa: E402
from test_gpu_chain_edges import assert_same, column_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

CARTPOLE3 = Kind("CartPole3", "CartPole", max_episode_steps=3)
CASES = ([(KINDS[k], p) for k in ("CartPole", "Pendulum", "Acrobot", "MountainCar")
          for p in ("f64", "f32")] +
         [(CARTPOLE3, "f64"), (CARTPOLE3, "f32"), (KINDS["FrozenLake4"], "f64"),
          (KINDS["Catch"], "f64")])
SIZES = (64, 1000, 65536)    # 1000: the last CTA is partly empty at both CTA sizes
T = 23                       # action rows; chains wrap around the stream
CHAIN_K = (1, 2, 9, 40)


def poison(pool):
    import torch

    from envpool_b200._capi import _torch_view

    _torch_view(pool.outputs_device_ptr(), (pool.slab_bytes,), torch.uint8, 0).fill_(0xFF)
    torch.cuda.synchronize()


def chain_case(kind, precision, n):
    import torch

    rng = np.random.default_rng(5)
    acts = torch.from_numpy(np.ascontiguousarray(kind.actions(rng, (T, n)))).cuda()
    torch.cuda.synchronize()
    pools = {m: kind.pool(n, 0, 3, precision) for m in ("graph", "plain", "direct")}
    try:
        for p in pools.values():
            p.reset_device()
        t = 0
        for K in CHAIN_K:
            for rep in range(2):  # the second run of a (t0, K) chain replays its graph
                for p in pools.values():
                    poison(p)
                pools["graph"].step_many_device(acts, t, K, use_graph=True)
                pools["plain"].step_many_device(acts, t, K, use_graph=False)
                for k in range(K):
                    pools["direct"].step_device(acts[(t + k) % T])
                torch.cuda.synchronize()
                want = column_bytes(pools["direct"])
                ctx = f"{kind.name}-{precision} n={n} K={K} t0={t} run {rep}"
                assert_same(column_bytes(pools["graph"]), want, ctx + " captured")
                assert_same(column_bytes(pools["plain"]), want, ctx + " uncaptured")
            t += K
    finally:
        for p in pools.values():
            p.close()


def chains_main():
    block = os.environ.get("ENVPOOL_B200_STEP_BLOCK")
    for kind, precision in CASES:
        for n in SIZES:
            chain_case(kind, precision, n)
        print(f"  block {block} {kind.name}-{precision}: sizes {SIZES}", flush=True)
    print("OK chains", flush=True)


@pytest.mark.parametrize("block", [64, 128])
def test_chained_steps_store_what_direct_steps_store(block):
    """Classic kinds in both precisions, CartPole at max_episode_steps = 3, FrozenLake and
    Catch at 64, 1000 and 65536 envs through the B-thread step kernel: after captured,
    replayed and uncaptured chains of 1, 2, 9 and 40 steps into a slab filled with 0xFF, every
    output column equals the same steps launched one by one."""
    env = dict(os.environ, ENVPOOL_B200_STEP_BLOCK=str(block))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "chains"],
                         capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "OK chains" in out.stdout, out.stdout[-3000:]


if __name__ == "__main__":
    chains_main()
