"""GPU: the peer exchange (csrc/exchange.cuh, the push / wait / chain code of csrc/capi.cu) for
every env kind, world size, ring depth, CTA size and push grid, and through the timed exchange
chain bench.py reports at N > 1.  Every rank's gathered batch is compared byte for byte with
un-exchanged twin pools after every call, and the twins with the oracle (tests/exchange_cases.py).

Direct exchanged steps run here, all ranks in this process: every rank's step has finished
before any wait is enqueued.  Chains and timed chains overlap the ranks' steps, pushes and waits
by design, so they run with one process per rank, attached through CUDA IPC as in the
one-process-per-GPU deployment (tests/exchange_matrix_check.py; exchange_cases.py says why),
one group of processes per setting of the variables the engine reads once per process or at
exchange_init, and one for the pushes of every kind's captured chains."""
import os
import subprocess
import sys

import pytest

from exchange_cases import CLASSIC, KINDS, PUSHED, Ranks

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))

# (kind, precision): every kind, the classic kinds in f32 as well.  push_kernel forwards the
# wire columns of every direct exchanged step, behind the step kernel on the same stream.
DIRECT = [(k, "f64") for k in KINDS] + [(k, "f32") for k in CLASSIC]


@pytest.fixture
def exchange_env(monkeypatch):
    """Leave no ENVPOOL_B200_EXCHANGE_DEPTH setting behind for the next test."""
    monkeypatch.delenv("ENVPOOL_B200_EXCHANGE_DEPTH", raising=False)
    return monkeypatch


@pytest.mark.parametrize("kind,precision", DIRECT, ids=[f"{k}-{p}" for k, p in DIRECT])
def test_direct_exchanged_steps_every_kind(capi, exchange_env, kind, precision):
    """W = 2, n = 1001 per rank (not a multiple of 4, 16 or 64: the wait kernel's tail quad,
    partial 16-byte units in push_kernel, a partial last step CTA), 40 steps
    with episodes short enough that envs reset through the exchange."""
    with Ranks(KINDS[kind], 1001, 2, precision=precision) as x:
        x.attach()
        x.reset()
        x.steps_direct(40)


@pytest.mark.parametrize("world", [1, 3, 4, 8, 16])
@pytest.mark.parametrize("kind", ["CartPole", "CliffWalkingSlippery"])
def test_world_sizes(capi, exchange_env, kind, world):
    """World sizes 1 .. 16 (kMaxPeers): rank g's constant id columns hold id0 + g * n + e in
    every slot of every rank, and every peer slice arrives (a record env and an RNG-in-step
    env, n = 257 per rank)."""
    with Ranks(KINDS[kind], 257, world) as x:
        x.attach()
        x.reset()
        x.steps_direct(12)


@pytest.mark.parametrize("world,n", [(2, 300_003), (4, 100_001)])
def test_wait_kernel_grid_stride_and_tail(capi, exchange_env, world, n):
    """More envs per rank than one pass of the wait kernel's capped grid covers (n / 4 >
    per_peer * 256 with per_peer = 2 * SMs / (W - 1)): the grid-stride loop runs, and n is
    not a multiple of 4, so the tail quad is re-expanded too.  The oracle checks the first and
    last 4096 envs and a strided sample."""
    with Ranks(KINDS["CartPole"], n, world) as x:
        x.attach()
        x.reset()
        x.steps_direct(10)


def test_128_thread_step_kernel_forwards_its_rows(capi, exchange_env):
    """Pendulum with 140,001 envs per rank is above 132 * 8 * 128, so the step kernel runs
    128-thread CTAs into its ring slot and push_kernel forwards the rows (bench.py's classic
    config at 2 GPUs has 524,288 per rank)."""
    with Ranks(KINDS["Pendulum"], 140_001, 2) as x:
        x.attach()
        x.reset()
        x.steps_direct(12)


def _group(group, **env):
    full = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32",
                ENVPOOL_B200_EXCHANGE_TIMEOUT_S="20")
    for k in ("EXCHANGE_DEPTH", "STEP_BLOCK", "PUSH_CTAS"):
        full.pop("ENVPOOL_B200_" + k, None)
    full.update({"ENVPOOL_B200_" + k: str(v) for k, v in env.items()})
    return subprocess.run([sys.executable, os.path.join(HERE, "exchange_matrix_check.py"), group],
                          capture_output=True, text=True, timeout=900, env=full)


def _run_group(group, **env):
    out = _group(group, **env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"OK {group}" in out.stdout, out.stdout[-3000:]


@pytest.mark.parametrize("depth", [2, 3, 5, 8])
@pytest.mark.parametrize("kind", ["CartPole", "Acrobot", "Taxi", "HalfCheetah"])
def test_ring_depths_direct_steps(capi, exchange_env, kind, depth):
    """ENVPOOL_B200_EXCHANGE_DEPTH = 2, 3, 5, 8 (read at exchange_init): direct exchanged steps
    through three wraps of the ring, so every slot's constant id columns, flags and per-slot
    step counters are used more than once."""
    exchange_env.setenv("ENVPOOL_B200_EXCHANGE_DEPTH", str(depth))
    with Ranks(KINDS[kind], 1001, 2) as x:
        x.attach()
        assert x.depth == depth
        x.reset()
        x.steps_direct(3 * depth + 1)


@pytest.mark.parametrize("depth", [2, 3, 4, 5, 8])
def test_chains_at_every_ring_depth_and_slot_phase(depth):
    """ENVPOOL_B200_EXCHANGE_DEPTH = 2, 3, 4 (the default), 5, 8 for CartPole, Acrobot, Taxi and
    HalfCheetah: captured and uncaptured chains of lengths
    1, D-1, D+1, 7, 2D, ... that start the next chain at every slot phase, more (K, phase) graph
    keys than the cache holds (evictions and recaptures), then a timed exchanged chain, direct
    exchanged steps and chains again."""
    _run_group(f"depth{depth}", EXCHANGE_DEPTH=depth)


@pytest.mark.parametrize("block", [128])
def test_step_kernel_cta_sizes(block):
    """ENVPOOL_B200_STEP_BLOCK = 128 (read once per process): the wider step kernel writes
    its ring slot before push_kernel forwards it, for rows of 12 (Pendulum, Blackjack obs),
    24 + 8 (Acrobot) and 100 bytes (Minesweeper's action mask), none a multiple of 16."""
    _run_group(f"block{block}", STEP_BLOCK=block)


@pytest.mark.parametrize("ctas", [1, 3])
def test_push_kernel_grids(ctas):
    """ENVPOOL_B200_PUSH_CTAS = 1 / 3 (read once per process): every push thread makes many
    passes over the wire columns (HalfCheetah, and CartPole's captured chains)."""
    _run_group(f"push{ctas}", PUSH_CTAS=ctas)


@pytest.fixture(scope="module")
def kinds_group():
    """The `kinds` group runs every case of the test below in one pair of processes."""
    return _group("kinds")


@pytest.mark.parametrize("kind,precision", PUSHED, ids=[f"{k.name}-{p}" for k, p in PUSHED])
def test_push_kernel_every_kind(kinds_group, kind, precision):
    """push_kernel on every kind's wire columns: captured exchanged chains of D + 1 steps put
    the pushes on branches beside the step chain, 40 steps with envs resetting through the
    exchange (direct steps push behind the step on its own stream instead)."""
    out = kinds_group
    assert out.returncode == 0 and f"kinds {kind.name}-{precision}: " in out.stdout, \
        out.stdout[-3000:] + out.stderr[-3000:]


def test_benchmark_shapes_through_the_timed_exchange_chain():
    """bench.py's N = 2 exchange path at its own shapes: plain chains, exchange_init / attach,
    a forced reset through the exchange, then step_many_timed(exchange=True) as Timer._one
    drives it (lead padded to a multiple of the ring depth, then once unpadded)."""
    _run_group("bench")
