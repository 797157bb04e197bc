"""GPU: the device RNG on CRAFTED engine states.

Sampled parity tests never reach the distribution branches that fire with probability
~2^-32 per draw: Lemire's rejection loop in uniform_int (Catch / FrozenLake: only the word 0;
Blackjack's range 13: nine words) and generate_canonical's `>= 1 -> nextafter(1, 0)` clamp.
tests/test_oracle_rng_vs_libstdcxx.py pins those branches of the ORACLE against libstdc++
itself on the CPU; here the same crafted states are loaded into the engine
(epb_state_import) and into the oracle (epo_debug_set_rng) and both must keep agreeing.

Crafting (toy_text_cases.crafted_table): a table whose words 0..8 are zero and whose words
397..404 are the untempered wanted outputs makes the next regeneration of chunk 0 (device:
mt_idx = 0; std::mt19937: position 624) emit exactly those outputs; every later chunk
regenerates identically on both sides because the whole 624-word table is the same."""
import numpy as np
import pytest

from helpers import assert_batch_equal
from toy_text_cases import crafted_table, load_both

pytestmark = pytest.mark.gpu


def patterns(rng, n, rejected):
    """Per env: 8 wanted outputs with rejected words sprinkled in (none, leading, doubled,
    trailing, all but one)."""
    out = []
    for e in range(n):
        w = [int(x) for x in rng.integers(1, 2**32, size=8)]
        r = lambda: int(rng.choice(rejected))  # noqa: E731
        kind = e % 6
        if kind == 1:
            w[0] = r()
        elif kind == 2:
            w[0] = w[1] = r()
        elif kind == 3:
            w[3] = r()
            w[7] = r()
        elif kind == 4:
            w = [r() for _ in range(7)] + [w[7]]
        elif kind == 5:
            w[1] = r()
            w[2] = r()
            w[5] = r()
        out.append(w)
    return out


@pytest.mark.parametrize("task,kw,n_act,rejected,force_done", [
    ("Catch", dict(), 3, [0], True),
    ("FrozenLake", dict(max_episode_steps=100, iopt=4), 4, [0], False),
    ("CliffWalking", dict(iopt=1), 4, [0], False),
    ("Blackjack", dict(iopt=2), 2, [(k * pow(13, -1, 2**32)) % 2**32 for k in range(9)], True),
    ("Taxi", dict(max_episode_steps=200), 6, [0], True),
])
def test_lemire_rejection_on_device(capi, task, kw, n_act, rejected, force_done):
    from oracle.oracle_lib import OraclePool

    n = 96
    rng = np.random.default_rng(11)
    pool = capi.CPool(task, n, seed=2, **kw)
    orc = OraclePool(task, n, seed=2, **kw)
    assert_batch_equal(pool.reset(), orc.reset(), task, 0.0, "reset")
    tables = np.stack([crafted_table(rng, w) for w in patterns(rng, n, rejected)])
    load_both(pool, orc, tables, force_done)
    for t in range(60):
        a = rng.integers(0, n_act, size=n).astype(np.int32)
        assert_batch_equal(pool.step(a), orc.step(a), task, 0.0, f"{task} t={t}")


def test_canonical_clamp_on_device(capi):
    from oracle.oracle_lib import OraclePool

    F = 0xFFFFFFFF
    n = 64
    rng = np.random.default_rng(5)
    for task, ms in (("CartPole", 500), ("Acrobot", 500)):
        pool = capi.CPool(task, n, seed=4, max_episode_steps=ms)
        orc = OraclePool(task, n, seed=4, max_episode_steps=ms)
        pool.reset()
        orc.reset()
        outs = []
        for e in range(n):
            w = [int(x) for x in rng.integers(0, 2**32, size=8)]
            if e % 4 == 0:
                w[0:4] = [F, F, 0, 0]              # canonical -> nextafter(1, 0), then 0.0
            elif e % 4 == 1:
                w[2:6] = [F, 0, 0, F]
            elif e % 4 == 2:
                w = [F] * 8
            outs.append(w)
        tables = np.stack([crafted_table(rng, w) for w in outs])
        load_both(pool, orc, tables, True)
        for t in range(30):
            a = rng.integers(0, 2, size=n).astype(np.int32)
            assert_batch_equal(pool.step(a), orc.step(a), task, 1e-6, f"{task} t={t}")
