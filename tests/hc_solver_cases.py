"""Crafted HalfCheetah states that drive the constraint solver through every branch, and the
branch traces that show it (test infrastructure).

The solver is the Newton loop of hc_pair_kernel (envpool_b200/csrc/mujoco_pair.cuh) and its
restatement in oracle/mjc_oracle.c.  Both record, under a test-only switch, every branch they
take (the HCP_STATS trace of the pair kernel's host build, tests/hc_pair_host/pair_stats.cc, and
mjc_solver_trace of the oracle); `parse` turns a trace into one record per mj_step and `branches`
names the branches a record took.  BRANCHES is the table the tests require to be covered.

`cases()` draws (q, v, qacc_warmstart, ctrl) candidates with a fixed seed, steps each once on the
host build of the pair kernel, and keeps those that take a branch fewer than PER_BRANCH kept states
have taken.  The candidate families:
  play      contacts of random play: folded legs near the floor, moderate speeds
  pressed   the torso 0.1 .. 0.2 into the floor, every leg joint past one end of its range
  extreme   speeds of 10 .. 1e6, ctrl far outside +-1, warm starts far off or the solver's answer
  free      high above the floor: no rows at all
  previous  a play / pressed state warm-started with the solver's own answer for it
  tie       a state warm-started with the host build's own qacc_smooth, bit for bit: cw == cs
  kink      a joint limit row exactly on the sj < 0 kink at the warm start (see `kink_case`)
The search tries SEARCH_BUDGET candidates whatever it has found; NOT_REACHED lists the branches it
does not reach with that budget.
"""
import ctypes
import functools
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "hc_pair_host", "pair_stats.cc")
SO = os.path.join(HERE, "hc_pair_host", "libhc_pair_stats.so")
HDRS = [os.path.join(ROOT, "envpool_b200", "csrc", f) for f in ("mujoco_pair.cuh", "mujoco_model.h")]

# trace events and values (mujoco_pair.cuh TR_*, mjc_oracle.c adds CONTACTS)
ROWS, WARM, LS, UPD, LS_END, EXIT, CONTACTS = range(1, 8)
RUN, SKIP_GS, SKIP_TOL = range(3)
NEWTON, EXPAND, BISECT = range(3)
CONV, STALL, CAP = range(3)
GRAD0, COST, GRAD, MAXITER, ALPHA0 = range(5)

# joint ranges of bthigh bshin bfoot fthigh fshin ffoot (half_cheetah.xml)
RANGE = np.array([[-.52, 1.05], [-.785, .785], [-.4, .785], [-1, .7], [-1.2, .87], [-.5, .5]])

BRANCHES = [
    ("rows 0", "no constraint row: free flight, qacc = qacc_smooth"),
    ("rows 1-9", "1 .. 9 merged rows in the two lanes"),
    ("rows 10-27", "10 .. 27 merged rows"),
    ("rows 28-54", "28 .. 54 merged rows"),
    ("warm kept", "cw < cs: qacc_warmstart kept"),
    ("warm smooth", "cw > cs: qacc_smooth taken"),
    ("warm tie", "cw == cs: qacc_warmstart kept"),
    ("exit grad0", "gradient test at iteration 0"),
    ("exit cost", "cost improvement below tolerance"),
    ("exit grad", "gradient test after an iteration"),
    ("exit max_iter", "iter == max_iter"),
    ("exit alpha0", "alpha == 0 after the line search"),
    ("ls skip gs", "line search skipped: !(gs < 0)"),
    ("ls skip gtol", "line search skipped: |gs| < gtol"),
    ("ls first", "converged at the first evaluation, alpha = 1"),
    ("ls newton", "a Newton update of alpha"),
    ("ls expand", "an expansion 2 alpha + 1 (hi = inf)"),
    ("ls bisect", "a bisection (lo + hi) / 2"),
    ("ls conv", "converged after at least one update"),
    ("ls stall", "next == alpha"),
    ("ls cap", "ls_iter evaluations without convergence"),
]
PER_BRANCH = 4
SEARCH_BUDGET = 2800
# Branches no candidate reaches within SEARCH_BUDGET (a search of 6000 found none either).
#  - exit max_iter: the Newton loop on this piecewise-quadratic cost ends within a few iterations.
#  - ls skip gtol, and with it exit alpha0 (the kernel's alpha is 0 only after a skipped search):
#    search = -H^-1 grad, so |gs| / |search| = g' H^-1 g / |H^-1 g|.  For it to fall below
#    gtol / |search| = 1e-10 / scale while scale |grad| >= 1e-8 (else the gradient test ends the
#    loop first), H must be conditioned worse than 4e4; this model's H stays near 1e4 or below
#    (pressed states, every contact active).  At speeds of 1e2 .. 1e7, where the gradient is
#    rounding noise, the loop ends on the cost test instead.
#  - ls skip gs: gs = -g' H^-1 g rounds to >= 0 (or is NaN) only for a far worse conditioned H.
NOT_REACHED = ("exit max_iter", "exit alpha0", "ls skip gs", "ls skip gtol")


@functools.lru_cache(maxsize=None)
def host():
    """The pair kernel's host build with the solver trace (built when stale)."""
    deps = [SRC] + HDRS
    if not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        subprocess.run(["g++", "-std=c++20", "-O2", "-fPIC", "-shared", "-pthread", "-w", SRC,
                        "-o", SO], check=True)
    H = ctypes.CDLL(SO)
    vp = ctypes.c_void_p
    H.hc_pair_host_step.argtypes = [ctypes.c_char_p, vp, vp, vp, vp, ctypes.c_int, ctypes.c_int]
    H.hc_pair_trace.argtypes = [ctypes.c_int, vp, ctypes.c_int]
    H.hc_pair_last_smooth.argtypes = [vp]
    return H


@functools.lru_cache(maxsize=None)
def model_blob():
    from envpool_b200 import _capi

    return _capi.hc_model_blob()


def host_step(state, ctrl, nsub=1, ks=27):
    """nsub mj_steps of the host build from state (q, v, w) [27]: (new state [27], trace of
    lane 0, trace of lane 1, qacc_smooth of the last mj_step)."""
    H = host()
    q, v, w = (np.array(state[i:i + 9], dtype=np.float64) for i in (0, 9, 18))
    a = np.ascontiguousarray(ctrl, dtype=np.float64)
    H.hc_pair_trace_clear()
    bad = H.hc_pair_host_step(model_blob(), q.ctypes.data, v.ctypes.data, w.ctypes.data,
                              a.ctypes.data, nsub, ks)
    assert bad == 0, "the duplicated root state of the two lanes is not bit-identical"
    tr = []
    for side in (0, 1):
        n = H.hc_pair_trace(side, None, 0)
        t = np.zeros(n, np.int32)
        H.hc_pair_trace(side, t.ctypes.data, n)
        tr.append(t)
    sm = np.zeros(9)
    H.hc_pair_last_smooth(sm.ctypes.data)
    return np.concatenate([q, v, w]), tr[0], tr[1], sm


class Oracle:
    """oracle/mjc_oracle.c on one state: one traced mj_step, or the constraint problem."""

    def __init__(self):
        from oracle.oracle_lib import MjcSim

        self.sim = MjcSim()
        L = self.sim.L
        for f in ("mjc_warm_mut", "mjc_ctrl_mut"):
            getattr(L, f).restype = ctypes.POINTER(ctypes.c_double)
            getattr(L, f).argtypes = [ctypes.c_void_p]
        L.mjc_solver_trace.argtypes = [ctypes.c_void_p, ctypes.c_int]
        self.L = L
        self.warm = np.ctypeslib.as_array(L.mjc_warm_mut(self.sim.d), shape=(9,))
        self.ctrl = np.ctypeslib.as_array(L.mjc_ctrl_mut(self.sim.d), shape=(6,))
        self.meaninertia = self.sim.constants()["meaninertia"]

    def _set(self, state, ctrl):
        self.sim.qpos[:], self.sim.qvel[:], self.warm[:] = state[:9], state[9:18], state[18:27]
        self.ctrl[:] = ctrl

    def step(self, state, ctrl, nsub=1):
        """(new state [27], trace) of nsub mj_steps."""
        self._set(state, ctrl)
        buf = np.zeros(1 << 16, np.int32)
        self.L.mjc_solver_trace(buf.ctypes.data, buf.size)
        self.sim.step(np.asarray(ctrl, dtype=np.float64), nsub)
        n = self.L.mjc_solver_trace(None, 0)
        assert n <= buf.size
        return np.r_[self.sim.qpos, self.sim.qvel, self.warm], buf[:n].copy()

    def problem(self, state, ctrl):
        """The constraint problem of the state's first mj_step, as the oracle's solver sees it:
        dict(M, qfrc_smooth, J, D, aref, qacc)."""
        self._set(state, ctrl)
        return self.sim.solve_problem()


def parse(trace):
    """A trace -> one record per mj_step: dict(rows, contacts, warm, ls=[dict(kind, upd, end)],
    exit).  Raises on an event out of order."""
    steps = []
    t = np.asarray(trace).reshape(-1, 2)
    for ev, val in t.tolist():
        if ev == ROWS:
            steps.append(dict(rows=val, contacts=None, warm=None, ls=[], exit=None))
            continue
        s = steps[-1]
        assert s["exit"] is None, ("event after the exit", ev, val)
        if ev == CONTACTS:
            s["contacts"] = val
        elif ev == WARM:
            assert s["warm"] is None and not s["ls"]
            s["warm"] = val
        elif ev == LS:
            s["ls"].append(dict(kind=val, upd=[], end=None))
        elif ev == UPD:
            assert s["ls"][-1]["end"] is None
            s["ls"][-1]["upd"].append(val)
        elif ev == LS_END:
            s["ls"][-1]["end"] = val
        elif ev == EXIT:
            s["exit"] = val
        else:
            raise AssertionError(("unknown event", ev, val))
    return steps


def oracle_as_kernel(step):
    """An oracle record in the pair kernel's terms.  The oracle writes 4 pyramid rows per contact,
    the kernel 3.  The oracle's line search evaluates alpha = 0 first, the kernel starts at
    alpha = 1 (phi''(0) = -phi'(0) makes the first Newton step land there): an oracle search whose
    first update is a Newton step from 0 is the kernel's search with that update dropped; one that
    converges at alpha = 0 is the kernel's |gs| < gtol skip; one that stalls at 0 (phi'(0) >= 0
    sets hi = 0) is the kernel's gs skip."""
    out = dict(step, rows=step["rows"] - (step["contacts"] or 0), contacts=None, ls=[])
    for s in step["ls"]:
        if not s["upd"] and s["end"] == CONV:
            out["ls"].append(dict(kind=SKIP_TOL, upd=[], end=None))
        elif not s["upd"] and s["end"] == STALL:
            out["ls"].append(dict(kind=SKIP_GS, upd=[], end=None))
        elif s["upd"][:1] == [NEWTON]:
            out["ls"].append(dict(kind=RUN, upd=s["upd"][1:], end=s["end"]))
        else:
            out["ls"].append(dict(s, kind=-1))   # no kernel counterpart: compares unequal
    return out


def branches(step):
    """The BRANCHES keys one kernel-terms record took."""
    b = set()
    r = step["rows"]
    b.add("rows 0" if r == 0 else "rows 1-9" if r < 10 else "rows 10-27" if r < 28 else
          "rows 28-54")
    if r == 0:
        return b
    w = step["warm"]
    b.add("warm tie" if w & 2 else "warm smooth" if w & 1 else "warm kept")
    b.add("exit " + {GRAD0: "grad0", COST: "cost", GRAD: "grad", MAXITER: "max_iter",
                     ALPHA0: "alpha0"}[step["exit"]])
    for s in step["ls"]:
        if s["kind"] != RUN:
            b.add("ls skip gs" if s["kind"] == SKIP_GS else "ls skip gtol")
            continue
        if not s["upd"] and s["end"] == CONV:
            b.add("ls first")
        elif s["end"] == CONV:
            b.add("ls conv")
        b.update("ls " + {NEWTON: "newton", EXPAND: "expand", BISECT: "bisect"}[u]
                 for u in s["upd"])
        if s["end"] == STALL:
            b.add("ls stall")
        if s["end"] == CAP:
            b.add("ls cap")
    return b


# ---------------------------------------------------------------------------------- search ---
def _play(rng):
    q = rng.uniform(-0.1, 0.1, 9)
    q[1] = rng.uniform(-0.25, 0.3)
    q[2] = rng.uniform(-1.5, 1.5)
    q[3:] = rng.uniform(-1.3, 1.3, 6)
    v = rng.normal(0, 2.0, 9)
    w = np.zeros(9) if rng.random() < 0.3 else rng.normal(0, 3.0, 9)
    return np.r_[q, v, w], rng.uniform(-1.2, 1.2, 6)


def _pressed(rng):
    q = np.zeros(9)
    q[0] = rng.uniform(-1, 1)
    q[1] = rng.uniform(-0.9, -0.8)
    q[2] = rng.uniform(-0.1, 0.1)
    past = rng.uniform(0.05, 0.4, 6)
    q[3:] = np.where(rng.random(6) < 0.5, RANGE[:, 0] - past, RANGE[:, 1] + past)
    return np.r_[q, rng.normal(0, 0.5, 9), rng.normal(0, 2.0, 9)], rng.uniform(-1.2, 1.2, 6)


def _extreme(rng):
    s, c = _play(rng) if rng.random() < 0.5 else _pressed(rng)
    s[9:18] = rng.normal(0, 10.0 ** rng.uniform(1, 6), 9)
    if rng.random() < 0.5:
        s[18:27] = rng.normal(0, 10.0 ** rng.uniform(0, 4), 9)
    else:
        s[18:27] = host_step(s, c)[0][18:27]
    return s, rng.uniform(-5, 5, 6)


def _free(rng):
    s, c = _play(rng)
    s[1] = rng.uniform(1.5, 3.0)
    return s, c


def _previous(rng):
    s, c = _play(rng) if rng.random() < 0.5 else _pressed(rng)
    s[18:27] = host_step(s, c)[0][18:27]
    return s, c


def _tie(rng):
    s, c = _play(rng) if rng.random() < 0.5 else _pressed(rng)
    s[18:27] = host_step(s, c)[3]
    return s, c


def kink_case(rng):
    """A joint pushed 0.05 .. 0.3 rad below its lower limit with zero joint speed, warm-started
    with the solver's answer except for that joint, whose warm acceleration is set to the limit
    row's aref.  The row's sj = 1 * w - aref is then exactly 0 at iteration 0 (its Jacobian is a
    single 1, the other products are exact zeros), in the kernel and in the oracle alike.  Past
    the impedance width the impedance is solimp_limit's dmax, so aref = -K dmax dist with K as
    fill_impedance_constants computes it, and with zero speed the damping term is an exact zero."""
    s, c = _pressed(rng)
    j = int(rng.integers(6))
    s[3 + j] = RANGE[j, 0] - rng.uniform(0.05, 0.3)
    s[12 + j] = 0.0
    s[18:27] = host_step(s, c)[0][18:27]
    hi, ref0, ref1 = 0.8, 0.02, 1.0
    K = 1.0 / (hi * hi * ref0 * ref0 * ref1 * ref1)
    dist = s[3 + j] - RANGE[j, 0]
    s[21 + j] = -0.0 - K * hi * dist
    return s, c


FAMILIES = ("play", "pressed", "extreme", "free", "previous", "tie", "kink")


@functools.lru_cache(maxsize=None)
def cases(seed=2024):
    """Crafted states: dict(states [N, 27], ctrl [N, 6], family [N] (names), hits [N] (sets of
    BRANCHES keys), counts {branch: states that took it}, tried)."""
    rng = np.random.default_rng(seed)
    gens = {"play": _play, "pressed": _pressed, "extreme": _extreme, "free": _free,
            "previous": _previous, "tie": _tie, "kink": kink_case}
    keys = [k for k, _ in BRANCHES]
    counts = dict.fromkeys(keys, 0)
    states, ctrls, fams, hits = [], [], [], []
    tried = 0
    # the kink and tie families exist for the branch they take by construction: keep a few of
    # each whatever else they take
    forced = {"kink": PER_BRANCH, "tie": PER_BRANCH}
    while tried < SEARCH_BUDGET:
        fam = FAMILIES[tried % len(FAMILIES)]
        tried += 1
        s, c = gens[fam](rng)
        _, t0, _, _ = host_step(s, c)
        rec = parse(t0)
        assert len(rec) == 1
        b = branches(rec[0])
        keep = any(counts[k] < PER_BRANCH for k in b)
        if fam in forced and forced[fam] > 0 and (fam != "kink" or "warm kept" in b):
            forced[fam] -= 1
            keep = True
        if keep:
            states.append(s)
            ctrls.append(c)
            fams.append(fam)
            hits.append(b)
            for k in b:
                counts[k] += 1
    return dict(states=np.array(states), ctrl=np.array(ctrls), family=fams, hits=hits,
                counts=counts, tried=tried)


def branch_table(c):
    """The branch table of cases() as text."""
    lines = [f"{'branch':14s} {'states':>6s}  meaning"]
    for k, d in BRANCHES:
        n = c["counts"][k]
        got = f"{n:6d}" if n else f"not reached, budget {c['tried']} candidates"
        lines.append(f"{k:14s} {got}  {d}")
    return "\n".join(lines)


# ------------------------------------------------------------- extended-precision minimiser ---
def mp_minimiser(p, dps=50):
    """The exact minimiser of the problem p (Oracle.problem) in mpmath at `dps` digits:
        cost(a) = 1/2 (a - a_s)' M (a - a_s) + sum_i 1/2 D_i min(0, J_i a - aref_i)^2,
    M a_s = qfrc_smooth.  Newton with exact line search: from the current point, the minimiser x
    of the quadratic piece whose active set (J_i a < aref_i) the point is on; if x is on the same
    piece it is the minimiser, otherwise the exact minimiser of cost on the ray towards x (phi' is
    piecewise linear: walk its breakpoints) is the next point.  Returns (a* as mpf list, cost
    function, gradient function), the functions taking float or mpf vectors."""
    import mpmath as mp

    mp.mp.dps = dps
    n = len(p["D"])
    M = mp.matrix(p["M"].tolist())
    fs = mp.matrix(p["qfrc_smooth"].tolist())
    J = [[mp.mpf(x) for x in row] for row in p["J"].tolist()]
    D = [mp.mpf(x) for x in p["D"].tolist()]
    aref = [mp.mpf(x) for x in p["aref"].tolist()]
    a_s = mp.lu_solve(M, fs)

    def vec(a):
        return mp.matrix([mp.mpf(x) for x in a]) if not isinstance(a, mp.matrix) else a

    def resid(a):
        return [mp.fsum(J[i][k] * a[k] for k in range(9)) - aref[i] for i in range(n)]

    def cost(a):
        a = vec(a)
        da = a - a_s
        r = resid(a)
        return (mp.fdot(da, M * da) / 2 +
                mp.fsum(D[i] * r[i] ** 2 for i in range(n) if r[i] < 0) / 2)

    def grad(a):
        a = vec(a)
        g = M * (a - a_s)
        r = resid(a)
        for i in range(n):
            if r[i] < 0:
                for k in range(9):
                    g[k] += D[i] * r[i] * J[i][k]
        return g

    def dphi(a, d, jd, r, t):   # phi'(t) along a + t d
        v = mp.fdot(d, M * (a + t * d - a_s))
        return v + mp.fsum(D[i] * (r[i] + t * jd[i]) * jd[i] for i in range(n)
                           if r[i] + t * jd[i] < 0)

    a = vec(p["qacc"])
    for _ in range(200):
        r = resid(a)
        act = [x < 0 for x in r]
        H, rhs = M.copy(), fs.copy()
        for i in range(n):
            if act[i]:
                for k in range(9):
                    rhs[k] += D[i] * aref[i] * J[i][k]
                    for m in range(9):
                        H[k, m] += D[i] * J[i][k] * J[i][m]
        x = mp.lu_solve(H, rhs)
        rx = resid(x)
        if all((rx[i] <= 0) if act[i] else (rx[i] >= 0) for i in range(n)):
            a = x
            break
        d = x - a
        jd = [mp.fsum(J[i][k] * d[k] for k in range(9)) for i in range(n)]
        bps = sorted(set(-r[i] / jd[i] for i in range(n) if jd[i] != 0 and -r[i] / jd[i] > 0))
        lo = mp.mpf(0)
        for hi in bps + [None]:
            # phi' is linear on [lo, hi]: its active set is the one at the midpoint
            mid = lo + 1 if hi is None else (lo + hi) / 2
            c1 = mp.fdot(d, M * d) + mp.fsum(D[i] * jd[i] ** 2 for i in range(n)
                                             if r[i] + mid * jd[i] < 0)
            c0 = dphi(a, d, jd, r, mid) - c1 * mid
            t = -c0 / c1
            if hi is None or t <= hi:
                break
            lo = hi
        a = a + max(t, lo) * d
    else:
        raise AssertionError("the extended-precision minimiser did not settle")
    return [a[k] for k in range(9)], cost, grad
