"""Body of the subprocess groups of tests/test_gpu_exchange_kinds.py: exchanged chains, timed
exchanged chains and the settings the engine reads once per process.  Run as

    CUDA_DEVICE_MAX_CONNECTIONS=32 ENVPOOL_B200_EXCHANGE_TIMEOUT_S=20 [ENVPOOL_B200_...=...] \
        python tests/exchange_matrix_check.py <group>

with group one of depth<D> (ENVPOOL_B200_EXCHANGE_DEPTH=D), block<B> (ENVPOOL_B200_STEP_BLOCK=B),
push<C> (ENVPOOL_B200_PUSH_CTAS=C), kinds or bench.  The command starts one process per rank
(W = 2, the same command with --rank r) on device 0; they meet in a gloo group and attach to
each other's gather buffers through CUDA IPC, as the one-process-per-GPU deployment does
(exchange_cases.py says why one process cannot play both ranks of an overlapped chain).  Each rank checks its own
gathered batch against all W twins after every call, rank 0 the twins against the oracle;
prints `OK <group>` when both ranks finished."""
import os
import socket
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from exchange_cases import BENCH_KINDS, KINDS, PUSHED, Ranks  # noqa: E402

WORLD = 2


def say(rank, msg):
    if rank == 0:
        print(msg, flush=True)


def depth_group(D, rank):
    """Chains of lengths 1, D-1, D+1, 7, 2D, ... move the next chain through the slot phases;
    the (K, phase) keys outnumber the 8 cached graphs, so captures are evicted and redone."""
    for name in ("CartPole", "Acrobot", "Taxi", "HalfCheetah"):
        with Ranks(KINDS[name], 1001, WORLD, rank=rank) as x:
            x.attach()
            assert x.depth == D, (x.depth, D)
            x.reset()
            keys = set()
            for K in (1, D - 1, D + 1, 7, 2 * D, 3, 2, 5, 1, 4, 6):
                keys.add(x.chain(K, use_graph=True))
            for K in (D + 1, 3):
                x.chain(K, use_graph=False)
            x.timed(5, D + 2)
            x.steps_direct(3)
            for K in (1, D - 1, D + 1, 7, 2, 3):
                keys.add(x.chain(K, use_graph=True))
            assert len({(K, phase) for K, _, phase in keys}) > 8, keys
        say(rank, f"  depth {D} {name}: {x.steps} steps")


def block_group(B, rank):
    """The B-thread step kernel writing its ring slot before push_kernel forwards it (every
    pool here runs that kernel, twins too)."""
    for name in ("Pendulum", "Acrobot", "Blackjack", "Minesweeper"):
        with Ranks(KINDS[name], 1001, WORLD, rank=rank) as x:
            x.attach()
            x.reset()
            x.steps_direct(8)
            x.chain(5, use_graph=True)
            x.chain(3, use_graph=False)
            x.steps_direct(2)
        say(rank, f"  block {B} {name}: {x.steps} steps")


def push_group(C, rank):
    """push_kernel with C CTAs: tens of passes per thread over the wire columns (every step of
    HalfCheetah, CartPole's steps in captured chains)."""
    for name, n in (("HalfCheetah", 4097), ("CartPole", 65537)):
        with Ranks(KINDS[name], n, WORLD, rank=rank) as x:
            x.attach()
            x.reset()
            x.steps_direct(4)
            x.chain(x.depth + 1, use_graph=True)
            x.chain(3, use_graph=False)
            x.timed(4, 4)
        say(rank, f"  push {C} {name}: {x.steps} steps")


def kinds_group(rank):
    """push_kernel on the wire columns of every kind: captured chains of D + 1 steps put each
    step's pushes on a branch beside the step chain, 40 steps in all, so that envs reset
    through the exchange.  Rank 0 prints one line per case."""
    for kind, precision in PUSHED:
        with Ranks(kind, 1001, WORLD, precision=precision, rank=rank) as x:
            x.attach()
            x.reset()
            while x.steps < 40:
                x.chain(x.depth + 1, use_graph=True)
        say(rank, f"  kinds {kind.name}-{precision}: {x.steps} steps")


# bench.py at --gpus 2: (kind, envs per rank, timed steps K, lead).  CartPole is the headline
# (lead = min(max(warmup, 128), 256)); the rest are run_config_line's BASELINE configs.
BENCH = [("CartPole", 65536, 64, 128), ("Pendulum", 1 << 19, 200, 32),
         ("Acrobot", 1 << 19, 100, 32), ("FrozenLake", 1 << 21, 100, 32),
         ("Catch", 1 << 21, 50, 32), ("HalfCheetah", 1 << 14, 10, 8)]


def bench_group(rank):
    """run_ours / run_config_line's sequence on one pool: plain chains and plain timed chains,
    exchange_init + attach, a forced reset through the exchange, then Timer._one's timed
    exchanged chains from action row 0 (lead padded so that lead + K is a multiple of the ring
    depth, the first replay warming the graph), then one unpadded chain and one padded chain
    at the new phase."""
    for name, n, K, lead in BENCH:
        with Ranks(BENCH_KINDS[name], n, WORLD, seed=0, T=8, rank=rank) as x:
            x.plain_reset()
            if name == "CartPole":   # warm-up launches, then replays of the same chain
                x.plain_chain(0, 16, use_graph=False)
                x.plain_chain(0, x.T, use_graph=True)
                x.plain_chain(0, x.T, use_graph=True)
            else:
                x.plain_chain(0, min(16, K))
            x.plain_timed(0, K, lead)
            x.plain_timed(0, K, lead)
            x.attach()
            x.reset()
            padded = lead + (-(lead + K)) % x.depth
            x.timed(K, padded, t0=0)
            x.timed(K, padded, t0=0)
            x.timed(K, lead, t0=0)
            x.timed(K, padded, t0=0)
        say(rank, f"  bench {name} x {n}: {x.steps} exchanged steps")


def run_rank(group, rank, port):
    from datetime import timedelta

    import torch
    import torch.distributed as dist

    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank,
                            world_size=WORLD, timeout=timedelta(seconds=300))
    if group.startswith("depth"):
        depth_group(int(group[5:]), rank)
    elif group.startswith("block"):
        block_group(int(group[5:]), rank)
    elif group.startswith("push"):
        push_group(int(group[4:]), rank)
    elif group == "kinds":
        kinds_group(rank)
    elif group == "bench":
        bench_group(rank)
    else:
        raise SystemExit(f"unknown group {group}")
    dist.barrier()
    dist.destroy_process_group()


def main(group):
    """Start the W rank processes, stop the others as soon as one fails, report."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    logs = [tempfile.TemporaryFile(mode="w+") for _ in range(WORLD)]
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), group, "--rank",
                               str(r), "--port", str(port)], stdout=logs[r],
                              stderr=subprocess.STDOUT) for r in range(WORLD)]
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
    print("OK", group)


if __name__ == "__main__":
    if "--rank" in sys.argv:
        run_rank(sys.argv[1], int(sys.argv[sys.argv.index("--rank") + 1]),
                 int(sys.argv[sys.argv.index("--port") + 1]))
    else:
        main(sys.argv[1])
