"""CPU: the crafted toy_text pools of toy_text_cases.py on the oracle alone.

test_gpu_toy_text.py compares the engine with the oracle on these pools.  A comparison is
only as strong as the branches its inputs reach, so this file asserts, on the oracle's own
outputs, that the crafted states and tables reach every branch the GPU test relies on: every
slip offset behind every rejection pattern, holes, goals and the time limit on one step, Taxi's
pickups and dropoffs, every Blackjack reward under every option, dealers that draw and bust,
both sides of NChain's 0.2 and every Catch catch and miss.  A table that stops reaching a
branch fails here instead of leaving the GPU test quietly weaker."""
import numpy as np
import pytest

import toy_text_cases as C
from helpers import assert_batch_equal, random_actions

TOY_VARIANTS = [("FrozenLake", 4, 100), ("FrozenLake", 8, 100), ("Catch", -1, -1),
                ("Taxi", -1, 200), ("NChain", -1, 1000), ("CliffWalking", 0, -1),
                ("CliffWalking", 1, -1)] + [("Blackjack", o, -1) for o in range(4)]


@pytest.mark.parametrize("k", [1, 8, 24, 200])
def test_crafted_table_forces_the_next_k_outputs(k):
    from oracle.oracle_lib import OraclePool

    rng = np.random.default_rng(k)
    want = rng.integers(0, 2**32, size=(16, k), dtype=np.uint64)
    want[:, 0] = [0, C.F] + [0x33333400] * 14
    tables = C.crafted_tables(rng, want)
    orc = OraclePool("NChain", 16, seed=0, max_episode_steps=1000)
    C.load_oracle(orc, tables)
    got = np.array([[orc.draw(e) for _ in range(k)] for e in range(16)], dtype=np.uint64)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("task,iopt,ms", TOY_VARIANTS)
def test_int_state_setter_round_trip(task, iopt, ms):
    """A free-running pool's integer states and RNG copied into a pool of another seed: both
    then step alike."""
    from oracle.oracle_lib import OraclePool

    n = 700
    rng = np.random.default_rng(3)
    a = OraclePool(task, n, seed=4, max_episode_steps=ms, iopt=iopt)
    b = OraclePool(task, n, seed=99, max_episode_steps=ms, iopt=iopt)
    a.reset()
    b.reset()
    for _ in range(37):
        a.step(random_actions(task, rng, (n,)))
    st = a.int_states()
    b.set_int_states(st)
    for e in range(n):
        b.set_rng(e, *a.rng(e))
    for k, v in b.int_states().items():
        assert np.array_equal(v, st[k]), k
    for t in range(40):
        act = random_actions(task, rng, (n,))
        assert_batch_equal(b.step(act), a.step(act), task, 0.0, f"{task} t={t}")
    for k, v in b.int_states().items():
        assert np.array_equal(v, a.int_states()[k]), k


def _moves(case, out0):
    """Rows whose first step moved the agent one cell: (row mask, move direction in the env's
    action numbering) from the start cell in the oracle state and the cell after step 1."""
    x0, y0 = case.ostate["i"][:, 0], case.ostate["i"][:, 1]
    width = case.iopt if case.task == "FrozenLake" else 12
    x1, y1 = out0["obs"] // width, out0["obs"] % width
    dx, dy = x1 - x0, y1 - y0
    if case.task == "FrozenLake":   # 0: --y, 1: ++x, 2: ++y, 3: --x
        table = {(0, -1): 0, (1, 0): 1, (0, 1): 2, (-1, 0): 3}
    else:                           # 0: --x, 1: ++y, 2: ++x, 3: --y
        table = {(-1, 0): 0, (0, 1): 1, (1, 0): 2, (0, -1): 3}
    d = np.array([table.get((int(a), int(b)), -1) for a, b in zip(dx, dy)])
    return d >= 0, d


def _check_slip_offsets(case, out0, valid=True):
    """Every first-step move must be the action turned by the offset the row's first
    accepted word gives, and every head pattern must show at least one move."""
    moved, d = _moves(case, out0)
    moved &= valid
    offset = (d - case.act0 + 1) % 4 - 1
    want = np.array([C.SLIP_OFFSET[int(w)] for w in
                     [next(v for v in row if v) for row in case.forced]])
    assert np.array_equal(offset[moved], want[moved])
    for h in range(len(C.SLIP_HEADS)):
        sel = moved & (case.heads == h)
        assert sel.any(), C.SLIP_HEADS[h]
    assert set(offset[moved].tolist()) == {-1, 0, 1}


def _frozen_lake(case, outs, _):
    o = outs[0]
    lake = C.LAKE4 if case.iopt == 4 else C.LAKE8
    cell = np.array([lake[v // case.iopt][v % case.iopt] for v in o["obs"]])
    _check_slip_offsets(case, o)
    hole, goal = (cell == "H") & o["done"], (cell == "G") & o["done"]
    assert hole.any() and goal.any()
    assert (o["reward"][goal] == 1).all() and (o["reward"][~goal] == 0).all()
    assert (o["trunc"] == (case.ostate["cur"] == 99)).all()       # the 100th step
    assert (hole & o["trunc"]).any() and (goal & o["trunc"]).any()
    assert (o["done"] & ~o["trunc"] & ~hole & ~goal).sum() == 0
    assert (o["trunc"] & ~hole & ~goal).any()


def _cliff(case, outs, _):
    o = outs[0]
    fell, goal = o["reward"] == -100, o["done"]
    assert fell.any() and goal.any()
    assert (o["obs"][fell] == 36).all() and (o["obs"][goal] == 47).all()
    if case.iopt:
        _check_slip_offsets(case, o, ~fell)


def _catch(case, outs, states):
    caught = {}
    for o, st in zip(outs, states):
        end = o["done"]
        for y, p, r in zip(st["i"][end, 1], st["i"][end, 2], o["reward"][end]):
            caught.setdefault(int(y), set()).add((int(y == p), float(r)))
    assert caught == {y: {(1, 1.0), (0, -1.0)} for y in range(5)}
    reset = case.ostate["done"] == 1
    assert (outs[0]["elapsed_step"][reset] == 0).all()
    assert set(states[0]["i"][reset, 1].tolist()) == set(range(5))   # every ball column


def _taxi(case, outs, states):
    o, st = outs[0], states[0]
    s0, s1 = case.ostate["i"][:, 2], st["i"][:, 2]
    pick, drop = case.act0 == 4, case.act0 == 5
    assert (pick & (o["reward"] == -1) & (s1 == 4)).any()            # pickup
    assert (pick & (o["reward"] == -10)).any()                       # no passenger here
    assert (drop & (o["reward"] == 20) & o["done"]).any()            # at the destination
    assert (drop & (o["reward"] == -1) & (s0 == 4) & (s1 < 4)).any()  # at another depot
    assert (drop & (o["reward"] == -10)).any()
    assert (o["trunc"] == (case.ostate["cur"] == 199)).all()
    assert (o["trunc"] & (o["reward"] == 20)).any()


def _nchain(case, outs, _):
    o = outs[0]
    s0 = case.ostate["i"][:, 0]
    # no slip: action 0 walks on (or earns 10 at the end), action 1 returns with 2
    stay = np.where(case.act0 == 0, np.where(s0 < 4, 0.0, 10.0), 2.0)
    slipped = o["reward"] != stay
    for h, (_, slips) in enumerate(C.NCHAIN_PAIRS):
        assert (slipped[case.heads == h] == slips).all(), C.NCHAIN_PAIRS[h]
    assert slipped.any() and (~slipped).any()
    assert (o["trunc"] == (case.ostate["cur"] == 999)).all()


def _bj_score(cards, n):
    raw = cards[:n].sum()
    s = raw + 10 if 1 in cards[:n] and raw + 10 <= 21 else raw
    return s


def _blackjack(cases_runs, option):
    natural, sab = option & 1, option >> 1
    rewards, long_dealer, dealer_bust = set(), False, False
    for case, (outs, states) in cases_runs:
        o, st = outs[0], states[0]
        rewards |= set(o["reward"].tolist())
        stick = case.act0 == 0
        long_dealer |= bool((st["ndealer"][stick] >= 5).any())
        dealer_bust |= any(_bj_score(st["dealer"][e], st["ndealer"][e]) > 21
                           for e in np.flatnonzero(stick)[:5000])
    want = {-1.0, 0.0, 1.0} | ({1.5} if natural and not sab else set())
    assert rewards == want
    assert long_dealer and dealer_bust


CHECKS = {"FrozenLake": _frozen_lake, "CliffWalking": _cliff, "Catch": _catch, "Taxi": _taxi,
          "NChain": _nchain}


@pytest.mark.parametrize("variant", C.VARIANTS)
def test_crafted_pools_reach_every_branch(variant):
    cases = C.builders()[variant]()
    for case in cases:
        assert case.n <= C.MAX_POOL
    runs = [(case, C.oracle_run(case)) for case in cases]
    if variant.startswith("Blackjack"):
        _blackjack(runs, cases[0].iopt)
        assert sum(c.n for c in cases) == (len(C.player_hands()) * 10 + 100 *
                                           len(C.PLAYER_PICKS)) * 2
    else:
        (case, (outs, states)), = runs
        CHECKS[case.task](case, outs, states)


def test_every_reachable_blackjack_hand_class():
    """(raw sum, ace, count, first two cards) of every hand a player can hold before a step."""
    hands = C.player_hands()
    assert len(hands) == 7456
    assert len({C._pack_hand(h) for h in hands}) == 7456
    assert all(sum(h) <= 21 for h in hands)

