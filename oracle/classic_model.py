"""TEST INFRASTRUCTURE ONLY: a host model of classic.cu's five classic_control steps, generic in
the state type R (np.float64 or np.float32), with the sin / cos values taken from a pluggable
provider.

In a classic step every operation other than sin / cos is an IEEE basic operation (+ - * /,
compares, casts), and classic.cu is compiled with -fmad=false, so none of them is contracted
into an FMA.  numpy's element-wise float64 / float32 operations are correctly rounded too.  The
model below does the engine's operations in the engine's order -- every constant cast as the
engine casts it, every literal an explicit R(...) -- and takes each sin / cos value from the
provider for the same argument, at the call site where the engine calls M<R>::sincos_small_,
sin_, cos_ or sincos_.  With the device provider (classic.cu's own functions, through
classic_lib) it must therefore reproduce the kernels bit for bit in both precisions; with the
libm provider the f64 model is the oracle's arithmetic (ep_oracle.c) bit for bit.

Every step also returns a record of which threshold, clip, wrap or goal branch fired, and the
intermediate values the crafted cases (tests/classic_cases.py) search on.
"""
from __future__ import annotations

import math

import numpy as np

TASKS = ("CartPole", "Pendulum", "Acrobot", "MountainCar", "MountainCarContinuous")
NR = {"CartPole": 4, "Pendulum": 2, "Acrobot": 4, "MountainCar": 2, "MountainCarContinuous": 2}


class LibmTrig:
    """libm's sin / cos (ep_oracle.c epo_trig) for every call site: the oracle's arithmetic."""

    name = "libm"

    @staticmethod
    def _both(x):
        from oracle.oracle_lib import libm_trig

        return libm_trig(np.asarray(x))

    def sincos_small(self, x):
        return self._both(x)

    def sincos(self, x):
        return self._both(x)

    def sin(self, x):
        from oracle.oracle_lib import libm_trig

        return libm_trig(np.asarray(x), want_cos=False)[0]

    def cos(self, x):
        from oracle.oracle_lib import libm_trig

        return libm_trig(np.asarray(x), want_sin=False)[1]


class DeviceTrig:
    """classic.cu's own M<R> functions on the current CUDA device (oracle/classic_lib.py)."""

    name = "device"

    def sincos_small(self, x):
        from oracle.classic_lib import device_trig

        return device_trig("sincos_small", x)

    def sincos(self, x):
        from oracle.classic_lib import device_trig

        return device_trig("sincos", x)

    def sin(self, x):
        from oracle.classic_lib import device_trig

        return device_trig("sin", x)[0]

    def cos(self, x):
        from oracle.classic_lib import device_trig

        return device_trig("cos", x)[1]


class HangRisk(ValueError):
    """An angle the engine's `while (theta >= pi) theta -= 2 pi` loops would not bring back into
    [-pi, pi) in reasonable time (infinite, NaN or huge)."""


def _wrap(theta, kPi):
    """while (theta < -kPi) theta += kPi * 2; while (theta >= kPi) theta -= kPi * 2;"""
    R = theta.dtype.type
    if not np.all(np.isfinite(theta)) or np.any(np.abs(theta) >= R(64 * math.pi)):
        raise HangRisk("angle not finite or beyond 64 pi before the wrap")
    theta = theta.copy()
    for up in (True, False):
        while True:
            m = theta < -kPi if up else theta >= kPi
            if not m.any():
                break
            theta[m] = theta[m] + kPi * R(2) if up else theta[m] - kPi * R(2)
    return theta


def _cols(s):
    return [np.array(s[:, k]) for k in range(s.shape[1])]


# ------------------------------------------------------------------------------ CartPole
def cartpole(R, trig, s, act):
    kGravity, kMassPole, kMassTotal = R(9.8), R(0.1), R(1.0 + 0.1)
    kLength, kMassPoleLength, kForceMag = R(0.5), R(0.1 * 0.5), R(10.0)
    kTau, kThetaThresholdRadians = R(0.02), R(12 * 2 * math.pi / 360)
    kXThreshold = R(2.4)
    x, x_dot, theta, theta_dot = _cols(s)
    force = np.where(np.asarray(act) == 1, kForceMag, -kForceMag).astype(R)
    sintheta, costheta = trig.sincos_small(theta)
    temp = (force + kMassPoleLength * theta_dot * theta_dot * sintheta) / kMassTotal
    theta_acc = ((kGravity * sintheta - costheta * temp) /
                 (kLength * (R(4.0 / 3.0) - kMassPole * costheta * costheta / kMassTotal)))
    x_acc = temp - kMassPoleLength * theta_acc * costheta / kMassTotal
    fallback = np.abs(theta) > R(0.5)   # the double sincos_small_ takes sincos() here
    x = x + kTau * x_dot
    x_dot = x_dot + kTau * x_acc
    theta = theta + kTau * theta_dot
    theta_dot = theta_dot + kTau * theta_acc
    br = {"x_lo": x < -kXThreshold, "x_hi": x > kXThreshold,
          "theta_lo": theta < -kThetaThresholdRadians, "theta_hi": theta > kThetaThresholdRadians,
          "x_eq_lo": x == -kXThreshold, "x_eq_hi": x == kXThreshold,
          "theta_eq_lo": theta == -kThetaThresholdRadians,
          "theta_eq_hi": theta == kThetaThresholdRadians,
          "sincos_small_fallback": fallback}
    term = br["x_lo"] | br["x_hi"] | br["theta_lo"] | br["theta_hi"]
    new = np.stack([x, x_dot, theta, theta_dot], 1)
    reward = np.full(len(x), 1.0, np.float32)
    aux = {"x": x, "theta": theta}
    return new, reward, term, br, aux


def cartpole_obs(R, trig, s):
    return {"obs": s.astype(np.float32)}


# ------------------------------------------------------------------------------ Pendulum
def pendulum(R, trig, s, act):
    kMaxSpeed, kMaxTorque, kDt, kGravity = R(8), R(2), R(0.05), R(10)
    kPi = R(math.pi)
    theta, theta_dot = _cols(s)
    act = np.asarray(act, np.float32).reshape(-1)
    u = act.astype(R)
    lo, hi = act < -kMaxTorque, act > kMaxTorque
    u = np.where(lo, -kMaxTorque, np.where(hi, kMaxTorque, u)).astype(R)
    cost = theta * theta + R(0.1) * theta_dot * theta_dot + R(0.001) * u * u
    new_theta_dot = theta_dot + R(3) * (kGravity / R(2) * trig.sin(theta) + u) * kDt
    theta = theta + new_theta_dot * kDt
    pre = theta
    vlo, vhi = new_theta_dot < -kMaxSpeed, new_theta_dot > kMaxSpeed
    theta_dot = np.where(vlo, -kMaxSpeed, np.where(vhi, kMaxSpeed, new_theta_dot)).astype(R)
    theta = _wrap(theta, kPi)
    br = {"u_lo": lo, "u_hi": hi, "u_eq_lo": act == -kMaxTorque, "u_eq_hi": act == kMaxTorque,
          "vel_lo": vlo, "vel_hi": vhi,
          "vel_eq_lo": new_theta_dot == -kMaxSpeed, "vel_eq_hi": new_theta_dot == kMaxSpeed,
          "wrap_up": pre < -kPi, "wrap_down": pre >= kPi,
          "theta_eq_neg_pi": pre == -kPi, "theta_eq_pi": pre == kPi}
    new = np.stack([theta, theta_dot], 1)
    reward = (-cost).astype(np.float32)
    aux = {"new_theta_dot": new_theta_dot, "theta": pre}
    return new, reward, np.zeros(len(theta), bool), br, aux


def pendulum_obs(R, trig, s):
    sn, cs = trig.sincos(np.array(s[:, 0]))
    return {"obs": np.stack([cs, sn, s[:, 1]], 1).astype(np.float32)}


# ------------------------------------------------------------------------------- Acrobot
def _derivs(R, trig, y):
    kG, kL, kM, kLC, kI = R(9.8), R(1), R(1), R(0.5), R(1)
    kHalfPi = R(math.pi / 2)
    theta1, theta2, dtheta1, dtheta2, a = y
    s2, c2 = trig.sincos(theta2)
    d1 = kM * kLC * kLC + kM * (kL * kL + kLC * kLC + R(2) * kL * kLC * c2) + kI * R(2)
    d2 = kM * (kLC * kLC + kL * kLC * c2) + kI
    phi2 = kM * kLC * kG * trig.cos(theta1 + theta2 - kHalfPi)
    phi1 = (-(dtheta2 + R(2) * dtheta1) * kM * kL * kLC * dtheta2 * s2 +
            kM * (kLC + kL) * kG * trig.cos(theta1 - kHalfPi) + phi2)
    ddtheta2 = ((a + d2 / d1 * phi1 - kM * kL * kLC * dtheta1 * dtheta1 * s2 - phi2) /
                (kM * kLC * kLC + kI - d2 * d2 / d1))
    ddtheta1 = -(d2 * ddtheta2 + phi1) / d1
    return [dtheta1, dtheta2, ddtheta1, ddtheta2, np.zeros_like(theta1)]


def _add(a, b):
    return [u + v for u, v in zip(a, b)]


def _mul(a, v):
    return [u * v for u in a]


def acrobot(R, trig, s, act):
    kPi, kMaxVel1, kMaxVel2 = R(math.pi), R(4 * math.pi), R(9 * math.pi)
    kDt = R(0.2)
    y0 = _cols(s) + [(np.asarray(act, np.int32) - 1).astype(R)]
    k1 = _derivs(R, trig, y0)
    k2 = _derivs(R, trig, _add(y0, _mul(k1, kDt / R(2))))
    k3 = _derivs(R, trig, _add(y0, _mul(k2, kDt / R(2))))
    k4 = _derivs(R, trig, _add(y0, _mul(k3, kDt)))
    total = _add(_add(_add(k1, _mul(k2, R(2))), _mul(k3, R(2))), k4)
    y = _add(y0, _mul(total, kDt / R(6.0)))
    pre = [v.copy() for v in y]
    y[0] = _wrap(y[0], kPi)
    y[1] = _wrap(y[1], kPi)
    br = {}
    for k in (0, 1):
        br[f"s{k}_wrap_up"] = pre[k] < -kPi
        br[f"s{k}_wrap_down"] = pre[k] >= kPi
        br[f"s{k}_eq_neg_pi"] = pre[k] == -kPi
        br[f"s{k}_eq_pi"] = pre[k] == kPi
    for k, lim in ((2, kMaxVel1), (3, kMaxVel2)):
        br[f"s{k}_lo"] = y[k] < -lim
        br[f"s{k}_hi"] = y[k] > lim
        y[k] = np.where(br[f"s{k}_lo"], -lim, y[k]).astype(R)
        y[k] = np.where(y[k] > lim, lim, y[k]).astype(R)
    # -cos_(s0) - cos_(s0 + s1) > 1
    height = -trig.cos(y[0]) - trig.cos(y[0] + y[1])
    term = height > R(1)
    br["height"] = term
    new = np.stack(y[:4], 1)
    reward = np.where(term, np.float32(0.0), np.float32(-1.0)).astype(np.float32)
    aux = {"s0": pre[0], "s1": pre[1], "height": height}
    return new, reward, term, br, aux


def acrobot_obs(R, trig, s):
    s0, c0 = trig.sincos(np.array(s[:, 0]))
    s1, c1 = trig.sincos(np.array(s[:, 1]))
    return {"obs": np.stack([c0, s0, c1, s1, s[:, 2], s[:, 3]], 1).astype(np.float32),
            "info:state": s[:, :2].astype(np.float32)}


# ------------------------------------------------------------------- MountainCar (+Cont.)
def _mountain_car(R, trig, s, action, continuous):
    kMinPos, kMaxPos, kMaxSpeed = R(-1.2), R(0.6), R(0.07)
    kGoalPos = R(0.45) if continuous else R(0.5)
    kGoalVel, kGravity = R(0), R(0.0025)
    pos, vel = _cols(s)
    br = {}
    if continuous:
        act = np.asarray(action, np.float32).reshape(-1).astype(R)
        reward = R(-0.1) * act * act
        br["act_lo"], br["act_hi"] = act < R(-1), act > R(1)
        br["act_eq_lo"], br["act_eq_hi"] = act == R(-1), act == R(1)
        act = np.where(br["act_lo"], R(-1), np.where(br["act_hi"], R(1), act)).astype(R)
        vel = vel + (act * R(0.0015) - trig.cos(R(3) * pos) * kGravity)
    else:
        act = (np.asarray(action, np.int32) - 1).astype(R)
        reward = np.full(len(pos), R(-1), R)
        vel = vel + (act * R(0.001) - trig.cos(R(3) * pos) * kGravity)
    pre_vel = vel
    br["vel_lo"], br["vel_hi"] = vel < -kMaxSpeed, vel > kMaxSpeed
    br["vel_eq_lo"], br["vel_eq_hi"] = vel == -kMaxSpeed, vel == kMaxSpeed
    vel = np.where(br["vel_lo"], -kMaxSpeed, np.where(br["vel_hi"], kMaxSpeed, vel)).astype(R)
    pos = pos + vel
    pre_pos = pos
    br["pos_lo"], br["pos_hi"] = pos < kMinPos, pos > kMaxPos
    br["pos_eq_min"] = pos == kMinPos
    pos = np.where(br["pos_lo"], kMinPos, np.where(br["pos_hi"], kMaxPos, pos)).astype(R)
    at_min = pos == kMinPos
    br["min_vel_neg"] = at_min & (vel < R(0))
    br["min_vel_zero"] = at_min & (vel == R(0))
    br["min_vel_pos"] = at_min & (vel > R(0))
    vel = np.where(br["min_vel_neg"], R(0), vel).astype(R)
    goal = (pos >= kGoalPos) & (vel >= kGoalVel)
    br["goal"] = goal
    br["goal_eq"] = (pos == kGoalPos) & (vel == R(0))
    br["below_goal_vel_zero"] = (pos < kGoalPos) & (vel == R(0))
    if continuous:
        reward = np.where(goal, reward + R(100), reward).astype(R)
    new = np.stack([pos, vel], 1)
    aux = {"vel": pre_vel, "pos": pre_pos}
    return new, reward.astype(np.float32), goal, br, aux


def mountain_car(R, trig, s, act):
    return _mountain_car(R, trig, s, act, False)


def mountain_car_continuous(R, trig, s, act):
    return _mountain_car(R, trig, s, act, True)


def mountain_car_obs(R, trig, s):
    return {"obs": s.astype(np.float32)}


STEP = {"CartPole": cartpole, "Pendulum": pendulum, "Acrobot": acrobot,
        "MountainCar": mountain_car, "MountainCarContinuous": mountain_car_continuous}
OBS = {"CartPole": cartpole_obs, "Pendulum": pendulum_obs, "Acrobot": acrobot_obs,
       "MountainCar": mountain_car_obs, "MountainCarContinuous": mountain_car_obs}


def step(task, R, trig, s, act):
    """One env step of every row of `s` ([n, NR] of R) under actions `act`: (new state,
    float32 reward, terminated, branch record, intermediates)."""
    s = np.ascontiguousarray(s, dtype=R)
    return STEP[task](R, trig, s, act)


def observe(task, R, trig, s):
    """The env-specific float32 output columns of states `s` (write_obs)."""
    return OBS[task](R, trig, np.ascontiguousarray(s, dtype=R))


def common(cur, done, max_steps):
    """The common columns as common.cuh's write_common computes them from the step counter and
    the done flag after the step."""
    cur = np.asarray(cur, np.int32)
    done = np.asarray(done, bool)
    return {"elapsed_step": cur, "done": done,
            "discount": np.where(done, np.float32(0), np.float32(1)).astype(np.float32),
            "step_type": np.where(cur == 0, 0, np.where(done, 2, 1)).astype(np.int32),
            "trunc": done & (cur >= max_steps)}


class ModelPool:
    """The engine's step of a whole pool (common.cuh env_step): rows whose done flag is set
    take their next initial state instead (reward 0, counter 0), every other row steps.
    `state` [n, NR] of R, `cur` and `done` per row."""

    def __init__(self, task, R, trig, state, cur, done, max_steps, env_ids=None):
        self.task, self.R, self.trig, self.max_steps = task, R, trig, max_steps
        self.state = np.array(state, dtype=R)
        self.cur = np.array(cur, np.int32)
        self.done = np.array(done, bool)
        n = len(self.cur)
        self.env_ids = np.arange(n, dtype=np.int32) if env_ids is None else np.asarray(
            env_ids, np.int32)
        self.branches = None

    def step(self, act, reset_state=None):
        """One step.  `reset_state(rows)` gives the next initial states ([len(rows), NR], any
        float type) of the rows that reset.  Returns the output columns."""
        R = self.R
        act = np.asarray(act)
        reset = self.done.copy()
        new, reward, term, br, _ = step(self.task, R, self.trig, self.state, act)
        cur = self.cur + 1
        done = (cur >= self.max_steps) | term
        rows = np.flatnonzero(reset)
        if rows.size:
            new[rows] = np.asarray(reset_state(rows)).astype(R)
            reward[rows] = np.float32(0)
            cur[rows] = 0
            done[rows] = False
        self.state, self.cur, self.done = new, cur.astype(np.int32), done
        self.branches = {k: v & ~reset for k, v in br.items()}
        out = common(self.cur, self.done, self.max_steps)
        out["reward"] = reward
        out["info:env_id"] = self.env_ids
        out["info:players.env_id"] = self.env_ids
        out.update(observe(self.task, R, self.trig, self.state))
        return out
