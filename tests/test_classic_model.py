"""CPU: the host model of classic.cu's steps (oracle/classic_model.py) with libm's sin / cos is
the oracle's arithmetic bit for bit, its crafted cases (classic_cases.py) reach every branch
boundary exactly in both precisions, and the hang guard refuses what could hang a GPU.

The GPU side (test_gpu_classic_model.py) holds the kernels to the same model fed the device's
own sin / cos; together the two pin the engine's f64 mode to the oracle up to the difference
between the device's and libm's sin / cos, which test_gpu_classic_model.py measures on its own."""
import numpy as np
import pytest

import classic_cases as C
from helpers import REGISTERED, random_actions
from oracle import classic_model as M

TRIG = M.LibmTrig()

# Every branch record key per env: each must fire on some crafted row and stay off on another,
# in both precisions.  *_eq_* keys are the exact boundaries.
BRANCHES = {
    "CartPole": {"x_lo", "x_hi", "theta_lo", "theta_hi", "x_eq_lo", "x_eq_hi", "theta_eq_lo",
                 "theta_eq_hi", "sincos_small_fallback"},
    "Pendulum": {"u_lo", "u_hi", "u_eq_lo", "u_eq_hi", "vel_lo", "vel_hi", "vel_eq_lo",
                 "vel_eq_hi", "wrap_up", "wrap_down", "theta_eq_neg_pi", "theta_eq_pi"},
    "Acrobot": {"s0_wrap_up", "s0_wrap_down", "s0_eq_neg_pi", "s0_eq_pi", "s1_wrap_up",
                "s1_wrap_down", "s1_eq_neg_pi", "s1_eq_pi", "s2_lo", "s2_hi", "s3_lo", "s3_hi",
                "height"},
    "MountainCar": {"vel_lo", "vel_hi", "vel_eq_lo", "vel_eq_hi", "pos_lo", "pos_hi",
                    "pos_eq_min", "min_vel_neg", "min_vel_zero", "min_vel_pos", "goal", "goal_eq",
                    "below_goal_vel_zero"},
}
BRANCHES["MountainCarContinuous"] = BRANCHES["MountainCar"] | {"act_lo", "act_hi", "act_eq_lo",
                                                               "act_eq_hi"}


def bits_equal(got, want, ctx):
    for k, w in want.items():
        g = np.ascontiguousarray(got[k])
        w = np.ascontiguousarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape, (ctx, k, g.dtype, w.dtype, g.shape)
        if g.tobytes() != w.tobytes():
            bad = np.flatnonzero((g.view(np.uint8) != w.view(np.uint8)).reshape(len(g), -1)
                                 .any(axis=1))
            raise AssertionError(f"{ctx} {k}: rows {bad[:5].tolist()} got "
                                 f"{g[bad[:3]].tolist()} want {w[bad[:3]].tolist()}")


def run_against_oracle(task, orc, model, acts, ctx):
    """Steps oracle and model on the same actions; every output column and the double state
    bit for bit after every step.  Rows that reset take the oracle's initial state."""
    nr = C.NR[task]
    for t, a in enumerate(acts):
        want = orc.step(a)
        st = orc.states()[:, :nr]
        got = model.step(a, lambda rows: st[rows])
        bits_equal(got, want, f"{ctx} t={t}")
        bits_equal({"state": model.state}, {"state": np.ascontiguousarray(st)}, f"{ctx} t={t}")


@pytest.mark.parametrize("task", C.CLASSIC)
def test_f64_model_equals_oracle_on_crafted_cases(task):
    """Every crafted case (found with libm's sin / cos) stepped by the oracle (state set with
    set_state) and by the f64 model: state, reward, flags and every output column bit for bit,
    on the crafted step and 12 free-running steps after it."""
    from oracle.oracle_lib import OraclePool

    case = C.build(task, np.float64, TRIG)
    ms, iopt = REGISTERED[task]
    orc = OraclePool(task, case.n, seed=3, max_episode_steps=ms, iopt=iopt)
    orc.reset()
    for e in range(case.n):
        s5 = np.zeros(5)
        s5[:C.NR[task]] = case.state[e]
        orc.set_state(e, s5, 0, int(case.cur[e]))
    model = M.ModelPool(task, np.float64, TRIG, case.state, case.cur, np.zeros(case.n, bool), ms)
    acts = np.concatenate([case.act[None],
                           random_actions(task, np.random.default_rng(1), (12, case.n))
                           .reshape((12,) + case.act.shape)])
    run_against_oracle(task, orc, model, acts, f"{task} crafted")


@pytest.mark.parametrize("task", C.CLASSIC)
def test_f64_model_equals_oracle_free_running(task):
    """2048 envs, 300 steps per env from the oracle's initial states, auto-resets included."""
    from oracle.oracle_lib import OraclePool

    n, T = 2048, 300
    ms, iopt = REGISTERED[task]
    orc = OraclePool(task, n, seed=7, max_episode_steps=ms, iopt=iopt)
    orc.reset()
    model = M.ModelPool(task, np.float64, TRIG, orc.states()[:, :C.NR[task]],
                        np.zeros(n, np.int32), np.zeros(n, bool), ms)
    acts = random_actions(task, np.random.default_rng(2), (T, n))
    run_against_oracle(task, orc, model, acts, f"{task} free-running")


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("task", C.CLASSIC)
def test_crafted_cases_reach_every_branch_boundary(task, precision):
    """Every threshold, clip, wrap and goal branch fires on some crafted row and not on
    another, and every exact-boundary case lands on its boundary (the *_eq_* keys)."""
    R = np.float64 if precision == "f64" else np.float32
    case = C.build(task, R, TRIG)
    br = M.step(task, R, TRIG, case.state, case.act)[3]
    assert set(br) == BRANCHES[task], sorted(set(br) ^ BRANCHES[task])
    never = sorted(k for k, v in br.items() if not v.any())
    always = sorted(k for k, v in br.items() if v.all())
    assert not never and not always, (never, always)
    for label in set(case.labels):
        if "exact" in label or "+0ulp" in label:
            rows = [i for i, lb in enumerate(case.labels) if lb == label]
            assert rows, label


def _case(task, R, state, act):
    n = len(state)
    return C.Case(task, R, np.asarray(state, R), act, np.zeros(n, np.int32), ["t"] * n)


@pytest.mark.parametrize("R", [np.float64, np.float32])
def test_guard_refuses_states_that_could_hang_the_wraps(R):
    """An infinite angle, a huge angle and an oversized velocity are refused before any GPU
    sees them; the libm model itself refuses to wrap a huge angle."""
    f = np.float32
    bad = [("Pendulum", [[np.inf, 0.0]], f([0])), ("Pendulum", [[1e6, 0.0]], f([0])),
           ("Pendulum", [[0.0, 17.0]], f([0])), ("Pendulum", [[-np.inf, 0.0]], f([0])),
           ("Acrobot", [[np.inf, 0.0, 0.0, 0.0]], [1]), ("Acrobot", [[0.0, 1e6, 0.0, 0.0]], [1]),
           ("Acrobot", [[0.0, 0.0, 13.0, 0.0]], [1]), ("Acrobot", [[0.0, 0.0, 0.0, 30.0]], [1]),
           ("CartPole", [[0.0, 0.0, np.inf, 0.0]], [1]),
           ("MountainCar", [[np.nan, 0.0]], [1]), ("Pendulum", [[0.0, 0.0]], f([np.nan]))]
    for task, s, a in bad:
        with pytest.raises(ValueError):
            C.guard(_case(task, R, s, a))
    with pytest.raises(M.HangRisk):
        M.step("Pendulum", R, TRIG, np.array([[1e6, 0.0]], R), f([0]))
    C.guard(_case("Pendulum", R, [[2 * np.pi * 0.999, 16.0]], f([2])))
