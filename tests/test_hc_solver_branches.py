"""CPU: HalfCheetah's constraint solver (the Newton loop and exact line search of hc_pair_kernel,
envpool_b200/csrc/mujoco_pair.cuh) driven through its branches on crafted states
(tests/hc_solver_cases.py), against the oracle's restatement (oracle/mjc_oracle.c) and against an
extended-precision minimiser of the problem both claim to solve.

What the kernel's source is held to, through its host build (two threads playing the lane pair):
  - every branch of the table in hc_solver_cases.BRANCHES is taken by some crafted state, except
    the ones NOT_REACHED lists, and those are not taken (a stale list fails);
  - both lanes take the same branches, event for event;
  - on states the solver resolves in double precision it takes the oracle's branch sequence, up
    to the documented difference of its line search's start (hc_solver_cases.oracle_as_kernel),
    and the two states after the mj_step agree within RESOLVED_BAR;
  - on "extreme" states (speeds up to 1e6, where phi' in the line search is rounding noise and
    either solver's path through stalls, bisections and the ls_iter cap is decided by that
    noise) the row count and warm-start choice agree and the states within EXTREME_BAR;
  - the solver's answer lies within the solver's own tolerance of the exact minimum:
    scale * (cost(qacc) - cost*) <= tolerance, scale = 1 / (meaninertia * nv), tolerance 1e-8,
    and scale * |grad(qacc)| <= tolerance wherever it stopped on the gradient test.  cost* is
    found in mpmath at 50 digits, with the KKT residual checked at 1e-25.
PARITY UNPINNED against MuJoCo itself, as everywhere else (DESIGN.md section 3)."""
import numpy as np
import pytest

import hc_solver_cases as hc

TOL = 1e-8                 # the model's solver tolerance
RESOLVED_BAR = 2e-12       # host build vs oracle, relative-absolute; measured 2.6e-13
EXTREME_BAR = 5e-11        # measured 6.7e-12


@pytest.fixture(scope="module")
def crafted():
    return hc.cases()


@pytest.fixture(scope="module")
def oracle():
    return hc.Oracle()


def _relerr(g, w):
    return float(np.max(np.abs(g - w) / (1 + np.abs(w))))


def test_every_branch_is_reached(crafted):
    print("\n" + hc.branch_table(crafted))
    for k, _ in hc.BRANCHES:
        if k in hc.NOT_REACHED:
            assert crafted["counts"][k] == 0, f"{k} is reached now: take it off NOT_REACHED"
        else:
            assert crafted["counts"][k] >= 1, k
    assert crafted["tried"] == hc.SEARCH_BUDGET


def test_lanes_take_the_same_branches(crafted):
    for i, (s, c) in enumerate(zip(crafted["states"], crafted["ctrl"])):
        for nsub, ks in ((1, 27), (5, 9), (5, 0)):
            _, t0, t1, _ = hc.host_step(s, c, nsub, ks)
            assert t0.size and np.array_equal(t0, t1), (i, nsub, ks)


def test_host_build_takes_the_oracles_branches(crafted, oracle):
    worst = {"resolved": 0.0, "extreme": 0.0}
    for i, (s, c, fam) in enumerate(zip(crafted["states"], crafted["ctrl"], crafted["family"])):
        got, t0, _, _ = hc.host_step(s, c)
        want, tw = oracle.step(s, c)
        g, = hc.parse(t0)
        w, = (hc.oracle_as_kernel(r) for r in hc.parse(tw))
        assert g["rows"] == w["rows"], (i, fam)
        ctx = (i, fam, g, w)
        if fam == "tie":
            # the host build's own qacc_smooth as warm start: a tie, and the warm start is kept.
            # The oracle's qacc_smooth differs in the last bits, so it sees no tie.
            assert g["warm"] == 2 or g["rows"] == 0, ctx
            g = dict(g, warm=None)
            w = dict(w, warm=None)
        if fam == "extreme":
            assert g["warm"] == w["warm"], ctx
            err, bar = _relerr(got, want), EXTREME_BAR
        else:
            assert g == w, ctx
            err, bar = _relerr(got, want), RESOLVED_BAR
        assert err <= bar, (i, fam, err)
        key = "extreme" if fam == "extreme" else "resolved"
        worst[key] = max(worst[key], err)
    print(f"\nhost build vs oracle after one mj_step: worst rel err {worst}")


def test_kink_states_sit_on_the_kink(crafted, oracle):
    """The kink family: the warm start is kept and one joint-limit row has sj == 0 exactly at it,
    in the oracle's arithmetic (J_i w - aref_i with J_i a single 1)."""
    n = 0
    for s, c, fam in zip(crafted["states"], crafted["ctrl"], crafted["family"]):
        if fam != "kink":
            continue
        p = oracle.problem(s, c)
        r = p["J"] @ s[18:27] - p["aref"]
        lim = (p["J"] != 0).sum(1) == 1
        assert (r[lim] == 0).any()
        n += 1
    assert n >= hc.PER_BRANCH


def solver_gaps(states, ctrls, families, qaccs, exits, oracle):
    """scale * (cost(qacc) - cost*) and, where exits[i] is a gradient exit, scale * |grad(qacc)|,
    per state; asserts both within TOL and the minimiser's KKT residual within 1e-25.  Returns
    [(gap, grad or None)] (None for states without rows)."""
    import mpmath as mp

    scale = 1.0 / (oracle.meaninertia * 9)
    out = []
    for i, (s, c) in enumerate(zip(states, ctrls)):
        p = oracle.problem(s, c)
        if len(p["D"]) == 0:
            out.append(None)
            continue
        a, cost, grad = hc.mp_minimiser(p)
        assert scale * mp.norm(grad(a)) < mp.mpf("1e-25"), i
        cstar = cost(a)
        gap = float(scale * (cost(qaccs[i]) - cstar))
        assert gap <= TOL, (i, families[i], gap)
        gn = None
        if exits[i] in (hc.GRAD0, hc.GRAD):
            gn = float(scale * mp.norm(grad(qaccs[i])))
            assert gn <= TOL, (i, families[i], gn)
        out.append((gap, gn))
    return out


def test_solvers_reach_the_minimiser(crafted, oracle):
    S, C, F = crafted["states"], crafted["ctrl"], crafted["family"]
    host_q, host_x, orc_q, orc_x = [], [], [], []
    for s, c in zip(S, C):
        got, t0, _, _ = hc.host_step(s, c)
        host_q.append(got[18:27])
        host_x.append(hc.parse(t0)[0]["exit"])
        want, tw = oracle.step(s, c)
        orc_q.append(want[18:27])
        orc_x.append(hc.parse(tw)[0]["exit"])
    rows = []
    for name, q, x in (("host build", host_q, host_x), ("oracle", orc_q, orc_x)):
        res = solver_gaps(S, C, F, q, x, oracle)
        for k, _ in hc.BRANCHES:
            sel = [r for r, h in zip(res, crafted["hits"]) if r is not None and k in h]
            if sel:
                gaps = max(r[0] for r in sel)
                grads = [r[1] for r in sel if r[1] is not None]
                rows.append(f"{name:10s} {k:14s} {len(sel):3d} states  worst gap {gaps:.1e}" +
                            (f"  worst grad {max(grads):.1e}" if grads else ""))
    print("\nscaled cost gap to the mpmath minimiser (tolerance 1e-8), by branch:\n" +
          "\n".join(rows))
