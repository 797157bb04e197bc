"""GPU: the programmatic edges of captured step chains (csrc/capi.cu run_chain).  Inside an
engine-captured chain each step may start while the step before it drains; everything a step
reads or writes sits behind its griddepcontrol.wait, so results must not change.  A captured
chain with timing marks is held byte for byte to the same steps launched directly
(use_graph=False): every output column after the last step, and the exported state blob (flags,
state, mt19937 tables, record rings, rcons / rprod).  The chains run six refill periods
(refill_every = 8 by default), so refills beside the chain and their joins are crossed several
times; chain lengths are multiples of the refill period, where both paths leave the record
rings full.

The CTA size of the step kernel is read once per process (ENVPOOL_B200_STEP_BLOCK), so each
size runs in a subprocess of its own: `python tests/test_gpu_chain_edges.py chains`.  Captured
exchanged chains at world size 2 run one process per rank on device 0, attached through CUDA
IPC (tests/exchange_cases.py says why one process cannot play both ranks of a chain):
`python tests/test_gpu_chain_edges.py exchange`."""
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
from exchange_cases import KINDS, Ranks  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = ([(k, p) for k in ("CartPole", "Pendulum", "Acrobot", "MountainCar",
                           "MountainCarContinuous") for p in ("f64", "f32")] +
         [("FrozenLake4", "f64"), ("Catch", "f64"), ("Game2048", "f64")])
SIZES = (64, 1000, 65536)    # 1000: the last CTA is partly empty at both CTA sizes
T = 37                       # action rows; chains wrap around the stream
CHAINS = ((0, 48, 8, 40), (5, 48, 3, 47))   # (t0, K, mark0, mark1): the second replays the graph


def column_bytes(pool):
    """Every output column of the last step, rows [0, n), as bytes."""
    import torch

    from envpool_b200._capi import _torch_view

    slab = _torch_view(pool.outputs_device_ptr(), (pool.slab_bytes,), torch.uint8, 0)
    return {k.name: slab[k.offset:k.offset + k.row_bytes * pool.n].cpu().numpy()
            for k in pool.keys}


def assert_same(got, want, ctx):
    for name in want:
        a, b = got[name], want[name]
        if not np.array_equal(a, b):
            i = int(np.flatnonzero(a != b)[0])
            raise AssertionError(f"{ctx}: `{name}` differs first at byte {i}")


def chain_case(name, precision, n):
    import torch

    kind = KINDS[name]
    rng = np.random.default_rng(11)
    acts = torch.from_numpy(np.ascontiguousarray(kind.actions(rng, (T, n)))).cuda()
    graph, direct = kind.pool(n, 0, 7, precision), kind.pool(n, 0, 7, precision)
    try:
        for p in (graph, direct):
            p.reset_device()
        for t0, K, mark0, mark1 in CHAINS:
            assert graph.step_many_timed(acts, t0, K, mark0, mark1, False, True) > 0
            direct.step_many_timed(acts, t0, K, mark0, mark1, False, False)
            torch.cuda.synchronize()
            ctx = f"{name}-{precision} n={n} chain t0={t0} K={K}"
            assert_same(column_bytes(graph), column_bytes(direct), ctx + " outputs")
            assert_same({"state": graph.state_export()}, {"state": direct.state_export()},
                        ctx + " state blob")
    finally:
        graph.close()
        direct.close()


def chains_main():
    block = os.environ.get("ENVPOOL_B200_STEP_BLOCK")
    for name, precision in CASES:
        for n in SIZES:
            chain_case(name, precision, n)
        print(f"  block {block} {name}-{precision}: sizes {SIZES}", flush=True)
    print("OK chains", flush=True)


def exchange_rank(rank, port):
    """Rank `rank` of two: the same exchanged chains captured and launched directly, each pair
    of Ranks checked against its twins after every call, and the two held to each other."""
    from datetime import timedelta

    import torch
    import torch.distributed as dist

    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=2, timeout=timedelta(seconds=300))
    for n in (4097, 65536):
        with Ranks(KINDS["CartPole"], n, 2, rank=rank) as g, \
                Ranks(KINDS["CartPole"], n, 2, rank=rank) as d:
            for x in (g, d):
                x.attach()
                x.reset()
            for K, lead in ((24, None), (16, None), (16, 8)):
                if lead is None:
                    g.chain(K, use_graph=True)
                    d.chain(K, use_graph=False)
                else:
                    g.timed(K, lead, use_graph=True)
                    d.timed(K, lead, use_graph=False)
                ctx = f"exchanged CartPole n={n} K={K} lead={lead} rank {rank}"
                assert_same(g.gathered(g.slot_ptr(g.pools[rank])),
                            d.gathered(d.slot_ptr(d.pools[rank])), ctx + " gathered batch")
                assert_same({"state": g.pools[rank].state_export()},
                            {"state": d.pools[rank].state_export()}, ctx + " state blob")
        if rank == 0:
            print(f"  exchange n={n}: {g.steps} steps", flush=True)
    dist.barrier()
    dist.destroy_process_group()


def exchange_main():
    """Start both rank processes, stop the other as soon as one fails, report."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    logs = [tempfile.TemporaryFile(mode="w+") for _ in range(2)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "exchange", "--rank",
                               str(r), "--port", str(port)], stdout=logs[r],
                              stderr=subprocess.STDOUT) for r in range(2)]
    try:
        while any(p.poll() is None for p in procs):
            if any(p.returncode not in (None, 0) for p in procs):
                break
            time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    for r, log in enumerate(logs):
        log.seek(0)
        print(f"--- rank {r} (exit {procs[r].returncode})\n{log.read()[-4000:]}", flush=True)
    if any(p.returncode != 0 for p in procs):
        raise SystemExit(1)
    print("OK exchange", flush=True)


def _run(group, **env):
    full = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32",
                ENVPOOL_B200_EXCHANGE_TIMEOUT_S="20")
    for k in ("EXCHANGE_DEPTH", "STEP_BLOCK", "PUSH_CTAS", "REC_Q", "REFILL_EVERY"):
        full.pop("ENVPOOL_B200_" + k, None)
    full.update({"ENVPOOL_B200_" + k: str(v) for k, v in env.items()})
    out = subprocess.run([sys.executable, os.path.abspath(__file__), group],
                         capture_output=True, text=True, timeout=900, env=full)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"OK {group}" in out.stdout, out.stdout[-3000:]


@pytest.mark.parametrize("block", [64, 128])
def test_captured_chain_matches_direct_launches(block):
    """Classic kinds in both precisions, FrozenLake, Catch and Game2048 at 64, 1000 and 65536
    envs through the B-thread step kernel: a captured timed chain and its replay equal the same
    steps launched directly, outputs and state blob byte for byte."""
    _run("chains", STEP_BLOCK=block)


def test_captured_exchanged_chain_matches_direct_launches():
    """World size 2 on one device, CartPole at 4097 and 65536 envs: captured exchanged chains
    and a captured timed exchanged chain equal the same chains launched directly, gathered
    batch and state blob byte for byte (and each equals its un-exchanged twins)."""
    _run("exchange")


if __name__ == "__main__":
    if "--rank" in sys.argv:
        exchange_rank(int(sys.argv[sys.argv.index("--rank") + 1]),
                      int(sys.argv[sys.argv.index("--port") + 1]))
    elif sys.argv[1] == "chains":
        chains_main()
    else:
        exchange_main()
