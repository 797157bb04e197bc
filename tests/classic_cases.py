"""Crafted classic_control states on the branch boundaries of classic.cu's steps, built with the
host model of oracle/classic_model.py, and the draw table of every env's initial states.

Each boundary is crafted by searching a free input -- one that enters the step after its last
sin / cos, so the landing point moves monotonically with it -- by bisection over the input's
floating-point values until the model, with the trig provider at hand, lands exactly on the
boundary; the cases one ulp either side are kept as well.  The GPU tests craft with the device's
sin / cos, the CPU tests with libm's, so every exact case is exact where it is run.

No case carries a NaN (CUDA and x86 NaN payloads differ), and every case passes `guard` before
it can reach a GPU: the engine's angle wraps (`while (theta >= pi) theta -= 2 pi`) never end
for an infinite or huge angle.

One boundary is unreachable and has no case: MountainCar's vel' == -0.0 at kMinPos.  vel' = vel + (accel - cos(3 pos) * g) is -0.0 only when both terms
are -0.0, and cos(3 pos) * g is never zero; x + (-x) rounds to +0.0.  The cases hold vel' == +0.0
there instead, and the smallest positive vel' that still leaves pos' == kMinPos.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import classic_model as M

CLASSIC = M.TASKS
NR = M.NR
REGISTERED_STEPS = {"CartPole": 500, "Pendulum": 200, "Acrobot": 500, "MountainCar": 200,
                    "MountainCarContinuous": 999}
CONTINUOUS = ("Pendulum", "MountainCarContinuous")


class Draws:
    """Each env's i-th initial state, from an oracle pool stepped only by forced resets: after
    its (i+1)-th reset it holds the state the engine's ring keeps as record i (record 0 is what
    the engine's first forced reset consumes)."""

    def __init__(self, task, n, seed, iopt, env_seed=None):
        from oracle.oracle_lib import OraclePool

        self.orc = OraclePool(task, n, seed=seed, iopt=iopt, env_seed=env_seed)
        self.nr = NR[task]
        self.table = np.empty((0, n, self.nr))

    def upto(self, m):
        """[>= m, n, NR] float64: records 0 .. m-1 of every env."""
        grow = []
        for _ in range(m - self.table.shape[0]):
            self.orc.reset()
            grow.append(self.orc.states()[:, :self.nr])
        if grow:
            self.table = np.concatenate([self.table, np.stack(grow)])
        return self.table


# ------------------------------------------------------------------------ float ordering
_INT = {np.dtype(np.float64): np.int64, np.dtype(np.float32): np.int32}


def _ord(x):
    """Monotone integer image of floats (-0.0 and +0.0 both map to 0)."""
    x = np.asarray(x)
    it = _INT[x.dtype]
    b = x.view(it).astype(np.int64)
    mag = b & np.int64(np.iinfo(it).max)
    return np.where(b < 0, -mag, mag)


def _unord(o, R):
    it = _INT[np.dtype(R)]
    o = np.asarray(o, np.int64)
    b = np.where(o < 0, (-o) | (np.int64(1) << (8 * np.dtype(it).itemsize - 1)), o)
    return b.astype(np.uint64).astype(np.dtype(it).str.replace("i", "u")).view(R)


def ulps(x, k):
    """x moved by k ulps (k < 0: down), in x's own type."""
    x = np.asarray(x)
    return _unord(_ord(x) + k, x.dtype.type)


# ------------------------------------------------------------------------------- cases
class Case:
    """Rows of crafted (state, action, step counter) of one env kind in one precision; every
    row steps (done flag clear).  `labels` says what each row was crafted for."""

    def __init__(self, task, R, state, act, cur, labels):
        self.task, self.R = task, R
        self.state = np.ascontiguousarray(state, dtype=R)
        dt = np.float32 if task in CONTINUOUS else np.int32
        self.act = np.ascontiguousarray(act, dtype=dt)
        self.cur = np.ascontiguousarray(cur, dtype=np.int32)
        self.labels = list(labels)
        self.max_steps = REGISTERED_STEPS[task]
        assert len(self.state) == len(self.act) == len(self.cur) == len(self.labels)

    @property
    def n(self):
        return len(self.cur)

    @property
    def flags(self):
        return (self.cur << 1).astype(np.int32)


def _step(task, R, trig, state, act):
    return M.step(task, R, trig, state, act)


def search(task, R, trig, base, act, col, key, target, lo, hi):
    """Per row: the input value v in [lo, hi] (column `col` of the state) at which the model's
    intermediate aux[key] first reaches target[row] from below (aux[key] must not decrease as v
    grows).  Returns (states with v set, hit) where hit says aux[key] == target exactly; rows
    whose bracket does not enclose the target come back with hit False."""
    base = np.array(base, dtype=R)
    n = len(base)
    target = np.broadcast_to(np.asarray(target, R), (n,))
    lo_o = np.broadcast_to(_ord(np.asarray(lo, R)), (n,)).copy()
    hi_o = np.broadcast_to(_ord(np.asarray(hi, R)), (n,)).copy()

    def f(o):
        s = base.copy()
        s[:, col] = _unord(o, R)
        return _step(task, R, trig, s, act)[4][key]

    ok = (f(lo_o) < target) & (f(hi_o) >= target)
    while np.any(hi_o > lo_o + 1):
        mid = (lo_o >> 1) + (hi_o >> 1) + (lo_o & hi_o & 1)   # floor((lo + hi) / 2), no overflow
        go = f(mid) >= target
        hi_o = np.where(go, mid, hi_o)
        lo_o = np.where(go, lo_o, mid)
    s = base.copy()
    s[:, col] = _unord(hi_o, R)
    hit = ok & (f(hi_o) == target)
    return s, hit


def _wrappable(task, R, s, act):
    """The rows of (s, act) whose angles the libm model finds within 4 pi before the wrap (the
    rows `guard` accepts)."""
    aux = M.step(task, R, M.LibmTrig(), s, act)[4]
    return np.flatnonzero((np.abs(aux["s0"]) < R(4 * math.pi)) &
                          (np.abs(aux["s1"]) < R(4 * math.pi)))


def _rows(states, acts, curs, labels):
    return (np.concatenate(states), np.concatenate(acts), np.concatenate(curs), sum(labels, []))


def _around(R, t):
    """t one ulp below, t, t one ulp above."""
    t = np.asarray([t], R)
    return np.concatenate([ulps(t, -1), t, ulps(t, 1)])


def cartpole(R, trig, rng):
    S, A, C, L = [], [], [], []
    kX, kTh = R(2.4), R(12 * 2 * math.pi / 360)
    for col, key, lim, name in ((0, "x", kX, "x"), (2, "theta", kTh, "theta")):
        for sign in (1, -1):
            tg = _around(R, sign * lim)
            for act in (0, 1):
                b = np.zeros((3, 4), R)
                b[:, 0] = R(sign * 2.39) if col == 0 else R(sign * 1.0)
                b[:, 2] = R(sign * 0.2) if col == 2 else R(sign * 0.05)
                b[:, 1] = R(0.3)
                b[:, 3] = R(-0.4)
                vcol = col + 1   # x' = x + tau * x_dot, theta' = theta + tau * theta_dot
                s, hit = search("CartPole", R, trig, b, np.full(3, act), vcol, key, tg, R(-2),
                                R(2))
                assert hit.all(), (name, sign, act)
                S.append(s); A.append(np.full(3, act)); C.append(np.full(3, 7))
                L.append([f"{name}' at {'+' if sign > 0 else '-'}threshold {d}"
                          for d in ("-1ulp", "exact", "+1ulp")])
    # termination on the truncation step, and each alone
    ms = REGISTERED_STEPS["CartPole"]
    s = np.array([[2.399, 1.0, 0.0, 0.0], [0.0, 0.0, 0.01, 0.0], [-2.399, -1.0, 0.0, 0.0]], R)
    for cur, tag in ((ms - 1, "on the truncation step"), (5, "mid-episode")):
        S.append(s); A.append(np.array([1, 0, 0])); C.append(np.full(3, cur))
        L.append([f"x' beyond +2.4 {tag}", f"inside the thresholds {tag}",
                  f"x' beyond -2.4 {tag}"])
    # signed zeros in every component, both actions
    z = np.array([[(-1.0) ** ((m >> k) & 1) * 0.0 for k in range(4)] for m in range(16)], R)
    for act in (0, 1):
        S.append(z); A.append(np.full(16, act)); C.append(np.full(16, 3))
        L.append([f"signed zeros {m:04b} act {act}" for m in range(16)])
    # sincos_small's switch at |theta| = 0.5 (the double path falls back to sincos above it)
    th = np.concatenate([_around(R, 0.5), _around(R, -0.5)])
    s = np.zeros((6, 4), R)
    s[:, 2] = th
    s[:, 3] = R(0.3)
    for act in (0, 1):
        S.append(s); A.append(np.full(6, act)); C.append(np.full(6, 2))
        L.append([f"theta {t!r} act {act}" for t in th])
    # random live states
    s = rng.uniform(-0.2, 0.2, (32, 4)).astype(R)
    S.append(s); A.append(rng.integers(0, 2, 32)); C.append(rng.integers(0, 400, 32))
    L.append(["random"] * 32)
    return Case("CartPole", R, *_rows(S, A, C, L))


def pendulum(R, trig, rng):
    S, A, C, L = [], [], [], []
    kPi = R(math.pi)
    # theta = +-0 (sin exact): new_theta_dot at +-8 and one ulp either side
    for th in (R(0.0), R(-0.0)):
        for sign in (1, -1):
            tg = _around(R, sign * 8.0)
            b = np.zeros((3, 2), R)
            b[:, 0] = th
            act = np.full(3, np.float32(0.7 * sign), np.float32)
            s, hit = search("Pendulum", R, trig, b, act, 1, "new_theta_dot", tg, R(-16), R(16))
            assert hit.all(), (th, sign)
            S.append(s); A.append(act); C.append(np.full(3, 9))
            L.append([f"theta {th!r} theta_dot' at {sign * 8} {d}" for d in ("-1ulp", "exact",
                                                                               "+1ulp")])
    # theta' exactly -pi (stays) and pi (wraps), and their neighbours
    for sign in (1, -1):
        tg = _around(R, sign * kPi)
        b = np.zeros((3, 2), R)
        b[:, 0] = R(sign * 3.0)
        act = np.full(3, np.float32(-0.3), np.float32)
        s, hit = search("Pendulum", R, trig, b, act, 1, "theta", tg, R(-16), R(16))
        assert hit.all(), sign
        S.append(s); A.append(act); C.append(np.full(3, 11))
        L.append([f"theta' at {'+' if sign > 0 else '-'}pi {d}" for d in ("-1ulp", "exact",
                                                                           "+1ulp")])
    # actions on and around the torque clip, signed zeros, infinities
    two = np.float32(2)
    acts = np.array([two, -two, np.nextafter(two, np.float32(0)), np.nextafter(two, np.float32(3)),
                     np.nextafter(-two, np.float32(0)), np.nextafter(-two, np.float32(-3)),
                     np.float32(0.0), np.float32(-0.0), np.float32(np.inf),
                     np.float32(-np.inf)], np.float32)
    s = np.stack([rng.uniform(-3, 3, len(acts)), rng.uniform(-8, 8, len(acts))], 1).astype(R)
    S.append(s); A.append(acts); C.append(np.full(len(acts), 4))
    L.append([f"action {a!r}" for a in acts])
    # wraps in both directions and the velocity clip from random states
    s = np.stack([rng.uniform(-math.pi, math.pi, 48), rng.uniform(-8, 8, 48)], 1).astype(R)
    s[:8, 0], s[:8, 1] = R(3.1), R(7.5)
    s[8:16, 0], s[8:16, 1] = R(-3.1), R(-7.5)
    S.append(s); A.append(rng.uniform(-2.5, 2.5, 48).astype(np.float32))
    C.append(np.full(48, 198)); L.append(["random"] * 48)
    s = np.array([[0.0, 0.0]], R)
    S.append(s); A.append(np.zeros(1, np.float32)); C.append(np.array([199]))
    L.append(["truncation"])
    return Case("Pendulum", R, *_rows(S, A, C, L))


def acrobot(R, trig, rng):
    S, A, C, L = [], [], [], []
    kPi = R(math.pi)
    v1, v2 = 4 * math.pi, 9 * math.pi
    # velocities at, just inside and beyond the clip limits after the step
    n = 64
    s = np.stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-math.pi, math.pi, n),
                  rng.choice([-v1, -0.99 * v1, 0.99 * v1, v1], n),
                  rng.choice([-v2, -0.99 * v2, 0.99 * v2, v2], n)], 1).astype(R)
    a = rng.integers(0, 3, n)
    k = _wrappable("Acrobot", R, s, a)
    S.append(s[k]); A.append(a[k]); C.append(np.full(len(k), 20))
    L.append(["velocity limits"] * len(k))
    # each angle onto +-pi exactly (where the search finds it), from several starting states
    for k, key in ((0, "s0"), (1, "s1")):
        for sign in (1, -1):
            m = 48
            b = np.stack([rng.uniform(-1, 1, m), rng.uniform(-1, 1, m),
                          rng.uniform(-2, 2, m), rng.uniform(-2, 2, m)], 1).astype(R)
            b[:, 2 + k] = R(sign * 3.0)   # turning towards the wrap
            act = rng.integers(0, 3, m)
            lo, hi = (R(1.5), R(3.1)) if sign > 0 else (R(-3.8), R(-2.2))
            for d in (0, -1, 1):
                tg = ulps(np.full(m, sign * kPi, R), d)
                st, hit = search("Acrobot", R, trig, b, act, k, key, tg, lo, hi)
                keep = np.flatnonzero(hit)[:4]
                S.append(st[keep]); A.append(act[keep]); C.append(np.full(len(keep), 30))
                L.append([f"{key}' at {'+' if sign > 0 else '-'}pi {d:+d}ulp"] * len(keep))
    # both sides of the height test, wraps in both directions: random states
    n = 96
    s = np.stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-math.pi, math.pi, n),
                  rng.uniform(-v1, v1, n), rng.uniform(-v2, v2, n)], 1).astype(R)
    a = rng.integers(0, 3, n)
    k = _wrappable("Acrobot", R, s, a)
    S.append(s[k]); A.append(a[k]); C.append(rng.integers(0, 500, n)[k])
    L.append(["random"] * len(k))
    return Case("Acrobot", R, *_rows(S, A, C, L))


def _mountain_car(task, R, trig, rng):
    cont = task == "MountainCarContinuous"
    S, A, C, L = [], [], [], []
    kMin, kV = R(-1.2), R(0.07)
    goal = R(0.45) if cont else R(0.5)

    def acts(n, v=None):
        if cont:
            return np.full(n, np.float32(0.4 if v is None else v), np.float32)
        return np.full(n, 2 if v is None else v, np.int32)

    def term(pos, act):
        """accel - cos(3 pos) * g of each row, exactly as the step computes it."""
        s = np.stack([pos, np.zeros_like(pos)], 1)
        return M.step(task, R, trig, s, act)[4]["vel"]

    # vel' at +-kMaxSpeed and one ulp either side
    for sign in (1, -1):
        b = np.zeros((3, 2), R)
        b[:, 0] = R(-0.5)
        a = acts(3)
        s, hit = search(task, R, trig, b, a, 1, "vel", _around(R, sign * kV), R(-0.08), R(0.08))
        assert hit.all(), sign
        S.append(s); A.append(a); C.append(np.full(3, 40))
        L.append([f"vel' at {sign * 0.07} {d}" for d in ("-1ulp", "exact", "+1ulp")])
    # pos' exactly kMinPos with vel' < 0 (and one ulp either side)
    b = np.zeros((3, 2), R)
    b[:, 0] = R(-1.15)
    a = acts(3, -1.0 if cont else 0)
    s, hit = search(task, R, trig, b, a, 1, "pos", _around(R, kMin), R(-0.07), R(0.0))
    assert hit.all()
    S.append(s); A.append(a); C.append(np.full(3, 41))
    L.append([f"pos' at kMinPos with vel' < 0 {d}" for d in ("-1ulp", "exact", "+1ulp")])
    # pos == kMinPos and vel' == +0.0 exactly, and the smallest vel' > 0 that keeps pos' there
    a = acts(2)
    pos = np.full(2, kMin, R)
    v = -term(pos, a)
    v[1] = ulps(v[1:2], 1)[0]
    S.append(np.stack([pos, v], 1)); A.append(a); C.append(np.full(2, 42))
    L.append(["pos' at kMinPos with vel' == +0.0", "pos' at kMinPos with vel' > 0"])
    # pos' beyond kMinPos (clipped, vel zeroed) and beyond kMaxPos (clipped, goal)
    s = np.array([[-1.19, -0.05], [-1.2, -0.07], [0.59, 0.05], [0.6, 0.07]], R)
    S.append(s); A.append(np.concatenate([acts(2, -1.0 if cont else 0), acts(2, 1.0 if cont
                                                                                else 2)]))
    C.append(np.full(4, 43)); L.append(["pos' below kMinPos"] * 2 + ["pos' above kMaxPos"] * 2)
    # pos' == goal exactly with vel' == 0 exactly (vel = -(accel - cos(3 pos) g)), and one ulp
    # below the goal
    a = acts(2)
    pos = np.array([goal, ulps(np.array([goal]), -1)[0]], R)
    S.append(np.stack([pos, -term(pos, a)], 1)); A.append(a); C.append(np.full(2, 44))
    L.append(["pos' at the goal with vel' == 0", "pos' one ulp below the goal with vel' == 0"])
    # the goal on the truncation step
    s = np.array([[0.58, 0.05], [-0.5, 0.0]], R)
    S.append(s); A.append(acts(2)); C.append(np.full(2, REGISTERED_STEPS[task] - 1))
    L.append(["goal on the truncation step", "truncation"])
    if cont:
        one = np.float32(1)
        av = np.array([one, -one, np.nextafter(one, np.float32(0)),
                       np.nextafter(one, np.float32(2)), np.nextafter(-one, np.float32(0)),
                       np.nextafter(-one, np.float32(-2)), np.float32(np.inf),
                       np.float32(-np.inf), np.float32(0.0), np.float32(-0.0)], np.float32)
        s = np.stack([rng.uniform(-1.2, 0.6, len(av)), rng.uniform(-0.07, 0.07, len(av))],
                     1).astype(R)
        s[6] = (0.44, 0.01)   # +inf action into the goal: reward -inf + 100
        S.append(s); A.append(av); C.append(np.full(len(av), 45))
        L.append([f"action {x!r}" for x in av])
    n = 32
    s = np.stack([rng.uniform(-1.2, 0.6, n), rng.uniform(-0.07, 0.07, n)], 1).astype(R)
    S.append(s)
    A.append(rng.uniform(-1.5, 1.5, n).astype(np.float32) if cont else rng.integers(0, 3, n))
    C.append(rng.integers(0, 150, n)); L.append(["random"] * n)
    return Case(task, R, *_rows(S, A, C, L))


BUILDERS = {"CartPole": cartpole, "Pendulum": pendulum, "Acrobot": acrobot,
            "MountainCar": lambda R, t, g: _mountain_car("MountainCar", R, t, g),
            "MountainCarContinuous": lambda R, t, g: _mountain_car("MountainCarContinuous", R,
                                                                    t, g)}


def build(task, R, trig, seed=0):
    """The crafted case of `task` in precision R, its exact boundaries found with `trig`;
    checked by `guard` before it is returned."""
    case = BUILDERS[task](R, trig, np.random.default_rng(seed))
    guard(case)
    return case


# ------------------------------------------------------------------------------ guard
ANGLE_LIMITS = {"Pendulum": ((0, 2 * math.pi), (1, 16.0)),
                "Acrobot": ((0, 2 * math.pi), (1, 2 * math.pi), (2, 4 * math.pi),
                            (3, 9 * math.pi))}


PRE_WRAP = {"Pendulum": ("theta",), "Acrobot": ("s0", "s1")}


def guard(case):
    """Refuses (ValueError) a case that could hang the engine's angle wraps or carries a NaN:
    every state and action must be free of NaN, every state finite, Pendulum's and Acrobot's
    angles within 2 pi and their velocities within reach (Pendulum |theta_dot| <= 16, Acrobot
    4 pi and 9 pi), and the libm model's angles after the step, before the wrap, finite and
    within 4 pi."""
    if np.isnan(case.act.astype(np.float64)).any():
        raise ValueError(f"{case.task}: NaN action")
    if not np.isfinite(case.state.astype(np.float64)).all():
        raise ValueError(f"{case.task}: state not finite")
    for col, lim in ANGLE_LIMITS.get(case.task, ()):
        bad = np.flatnonzero(np.abs(case.state[:, col]) > case.R(lim))
        if bad.size:
            raise ValueError(f"{case.task}: state column {col} beyond {lim:g} at rows "
                             f"{bad[:5].tolist()}")
    try:
        aux = M.step(case.task, case.R, M.LibmTrig(), case.state, case.act)[4]
    except M.HangRisk as e:
        raise ValueError(f"{case.task}: {e}") from None
    for key in PRE_WRAP.get(case.task, ()):
        if not (np.abs(aux[key]) < case.R(4 * math.pi)).all():
            raise ValueError(f"{case.task}: {key} beyond 4 pi after the step")
    return case
