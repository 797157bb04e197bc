"""GPU: the toy_text family (envpool_b200/csrc/toytext.cu) bit for bit against the oracle on
every reachable state and action, in every compiled kernel and through every entry point.

Each env is instantiated into four kernels -- step_kernel<Env, 64 / 128 / 256> and
rollout_kernel<Env> -- that ptxas compiles one by one, so a miscompile can sit in one of them
alone (toytext.cu's CliffWalking note records one).  The crafted pools of toy_text_cases.py
(every reachable state x every action, mt19937 tables forced onto each draw's boundaries,
their coverage asserted by test_toy_text_crafted.py) go through each of them; long runs take
the device's chunked mt19937 through more than two table generations; and the benchmark's
4,194,304-env chains are checked on a sample of envs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import toy_text_cases as C
from helpers import REGISTERED, assert_batch_equal, random_actions

pytestmark = pytest.mark.gpu


def _torch_dtypes():
    import torch

    return {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
            np.dtype(np.bool_): torch.bool}


def eq(got, want, task, ctx):
    assert_batch_equal(got, want, task, 0.0, ctx)


def outputs(pool, rows=None):
    out = pool.outputs_torch()
    return {k: (v if rows is None else v[rows]).cpu().numpy() for k, v in out.items()}


def crafted_pool(capi, case):
    pool = capi.CPool(case.task, case.n, seed=0, **case.kwargs())
    pool.reset()
    C.load_engine(pool, case.tables, case.istate, case.flags)
    return pool


def check_state(case, blob_state, ostate, ctx):
    """The engine's packed words against the oracle's fields, env by env."""
    w = blob_state["istate"]
    o = ostate["i"]
    flags = blob_state["flags"]
    assert np.array_equal(flags & 1, ostate["done"]), (ctx, "done")
    assert np.array_equal(flags >> 1, ostate["cur"]), (ctx, "cur")
    if case.task == "Blackjack":
        for k, hand in ((0, "player"), (1, "dealer")):
            n = ostate["n" + hand]
            cards = np.where(np.arange(32) < n[:, None], ostate[hand], 0)  # a reset leaves cards
            got = np.stack([w[k] & 63, (w[k] >> 6) & 1, (w[k] >> 7) & 31, (w[k] >> 12) & 15,
                            (w[k] >> 16) & 15])
            want = np.stack([cards.sum(1), (cards == 1).any(1), n, cards[:, 0], cards[:, 1]])
            assert np.array_equal(got, want), (ctx, hand)
        return
    fields = {"FrozenLake": [(0, 7), (3, 7)], "Catch": [(0, 255), (8, 255), (16, 255)],
              "Taxi": [(0, 15), (4, 15), (8, 15), (12, 15)], "NChain": [(0, -1)],
              "CliffWalking": [(0, 255), (8, 255)]}[case.task]
    for j, (shift, mask) in enumerate(fields):
        assert np.array_equal((w[0] >> shift) & mask, o[:, j]), (ctx, j)


def host_path(capi, case, outs, last_state):
    """Crafted case through the host path (the step kernel step_block_for picks): every step's
    outputs and the final state words against the oracle.  Returns the exported state blob."""
    pool = crafted_pool(capi, case)
    for t, a in enumerate(case.actions()):
        eq(pool.step(a), outs[t], case.task, f"{case.name} host t={t}")
    blob = pool.state_export()
    check_state(case, pool.state_arrays(blob), last_state, case.name)
    pool.close()
    return blob


def run_variant_host_path(capi, variant):
    for case in C.builders()[variant]():
        outs, states = C.oracle_run(case, every_state=False)
        host_path(capi, case, outs, states[-1])


@pytest.mark.parametrize("variant", C.VARIANTS)
def test_crafted_states_through_every_entry_point(capi, variant):
    """Host path (the 64-thread step kernel at these sizes), the rollout kernel, and captured,
    direct and timed step chains, from the same crafted state: every output column of every
    step against the oracle, the engine's state words against the oracle's state, and the same
    state bytes from every path."""
    import torch

    for case in C.builders()[variant]():
        outs, states = C.oracle_run(case, every_state=False)
        acts = case.actions()
        d_acts = torch.from_numpy(acts).cuda()
        T, N = acts.shape
        blob = host_path(capi, case, outs, states[-1])

        roll = crafted_pool(capi, case)
        tdt = _torch_dtypes()
        cols = [torch.empty((T, N) + k.shape, dtype=tdt[k.dtype], device="cuda")
                for k in roll.keys]
        roll.rollout_device(d_acts, T, cols)
        roll.sync()
        for t in range(T):
            got = {k.name: c[t].cpu().numpy() for k, c in zip(roll.keys, cols)}
            eq(got, outs[t], case.task, f"{case.name} rollout t={t}")
        assert np.array_equal(roll.state_export(), blob), (case.name, "rollout state")
        del cols

        for how in ("graph", "direct", "timed"):
            p = crafted_pool(capi, case)
            if how == "timed":
                assert p.step_many_timed(d_acts, 0, T, 2, T) > 0
            else:
                p.step_many_device(d_acts, 0, T, use_graph=how == "graph")
            p.sync()
            eq(outputs(p), outs[-1], case.task, f"{case.name} {how} chain")
            assert np.array_equal(p.state_export(), blob), (case.name, how)
            p.close()


def test_catch_permuted_and_partial_batches(capi):
    """Catch writes its 10x5 grid block-cooperatively (block_write_obs): rows in a permuted
    order, and batches that end inside a CTA."""
    from oracle.oracle_lib import OraclePool

    case = C.catch()
    pool = crafted_pool(capi, case)
    orc = OraclePool(case.task, case.n, seed=0, **case.kwargs())
    C.load_oracle(orc, case.tables, case.ostate)
    rng = np.random.default_rng(12)
    for t in range(24):
        ids = rng.permutation(case.n).astype(np.int32)
        if t % 2:
            ids = ids[:int(rng.choice([1, 63, 65, 1001, case.n - 1]))]
        a = rng.integers(0, 3, size=len(ids)).astype(np.int32)
        eq(pool.step(a, ids), orc.step(a, ids), "Catch", f"t={t} batch={len(ids)}")


_BLOCK = """
import sys
from envpool_b200 import _capi
import test_gpu_toy_text as G
_capi.load_library()
for variant in G.C.VARIANTS:
    G.run_variant_host_path(_capi, variant)
print("BLOCK%s OK" % sys.argv[1])
"""


@pytest.mark.parametrize("block", [128, 256])
def test_crafted_states_on_the_wide_step_kernels_in_a_subprocess(capi, block):
    """ENVPOOL_B200_STEP_BLOCK is read once per process: a fresh interpreter steps every
    crafted pool on the 128- or 256-thread step kernel against the oracle."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, ENVPOOL_B200_STEP_BLOCK=str(block),
               PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]))
    r = subprocess.run([sys.executable, "-s", "-c", _BLOCK, str(block)], env=env, cwd=here,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and f"BLOCK{block} OK" in r.stdout, \
        r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.parametrize("task,iopt,ms,T", [("FrozenLake", 4, 100, 1300),
                                            ("FrozenLake", 8, 100, 1300),
                                            ("CliffWalking", 1, -1, 1300),
                                            ("NChain", -1, 1000, 700)])
def test_more_than_two_table_generations(capi, task, iopt, ms, T):
    """Each env draws at least 1248 words (NChain: two per step), so the device regenerates
    its table twice from words it wrote itself.  Rollout in pieces row by row; captured, direct
    and timed chains over the whole run."""
    import torch

    from oracle.oracle_lib import OraclePool

    N = 1001
    rng = np.random.default_rng(31)
    acts = random_actions(task, rng, (T, N))
    d_acts = torch.from_numpy(acts).cuda()
    orc = OraclePool(task, N, seed=17, max_episode_steps=ms, iopt=iopt)
    orc.reset()
    want = [orc.step(acts[t]) for t in range(T)]

    roll = capi.CPool(task, N, seed=17, max_episode_steps=ms, iopt=iopt)
    roll.reset_device()
    tdt = _torch_dtypes()
    t0 = 0
    for piece in (1, 400, T - 401):
        cols = [torch.empty((piece, N) + k.shape, dtype=tdt[k.dtype], device="cuda")
                for k in roll.keys]
        roll.rollout_device(d_acts[t0:t0 + piece].contiguous(), piece, cols)
        roll.sync()
        for t in range(piece):
            got = {k.name: c[t].cpu().numpy() for k, c in zip(roll.keys, cols)}
            eq(got, want[t0 + t], task, f"rollout t={t0 + t}")
        t0 += piece
    blob = roll.state_export()
    assert (roll.state_arrays(blob)["mt_idx"] != 0).any()

    for how in ("graph", "direct", "timed"):
        p = capi.CPool(task, N, seed=17, max_episode_steps=ms, iopt=iopt)
        p.reset_device()
        if how == "timed":
            assert p.step_many_timed(d_acts, 0, T, 8, T) > 0
        else:
            p.step_many_device(d_acts, 0, T, use_graph=how == "graph")
        p.sync()
        eq(outputs(p), want[-1], task, f"{how} chain")
        assert np.array_equal(p.state_export(), blob), how
        p.close()


@pytest.mark.parametrize("task,steps", [("FrozenLake", 100), ("Catch", 50)])
def test_benchmark_shape_chains(capi, task, steps):
    """bench.py's toy_text configs: 4,194,304 envs (the 128-thread step kernel), seed 0 and the
    registered limits; 16 warm-up steps of a captured chain, then the Timer's timed chains of 32
    lead-in + `steps` steps, each replayed twice, all reading a 64-row action stream from row 0.
    After each chain: the first and last 4096 envs and a strided sample against an oracle
    seeded seed + env id."""
    import torch

    from oracle.oracle_lib import OraclePool

    N, lead, seed = 1 << 22, 32, 0
    ms, iopt = REGISTERED[task]
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    d_acts = torch.randint(0, 4 if task == "FrozenLake" else 3, (64, N), generator=g,
                           device="cuda", dtype=torch.int32)
    ids = np.unique(np.concatenate([np.arange(4096), np.arange(N - 4096, N),
                                    np.arange(4096, N - 4096, 1021)])).astype(np.int32)
    d_ids = torch.from_numpy(ids).long().cuda()
    acts = d_acts[:, d_ids].cpu().numpy()
    pool = capi.CPool(task, N, seed=seed, max_episode_steps=ms, iopt=iopt)
    orc = OraclePool(task, len(ids), env_seed=ids + seed, max_episode_steps=ms, iopt=iopt)

    def check(want, ctx):
        want = dict(want, **{"info:env_id": ids, "info:players.env_id": ids})
        eq(outputs(pool, d_ids), want, task, ctx)

    pool.reset_device()
    pool.sync()
    check(orc.reset(), "reset")
    pool.step_many_device(d_acts, 0, 16)
    pool.sync()
    for k in range(16):
        want = orc.step(acts[k])
    check(want, "warm-up chain")
    n_chain = lead + steps
    for rep in range(2):
        assert pool.step_many_timed(d_acts, 0, n_chain, lead, n_chain) > 0
        for k in range(n_chain):
            want = orc.step(acts[k % 64])
        check(want, f"timed chain {rep}")
    pool.close()
