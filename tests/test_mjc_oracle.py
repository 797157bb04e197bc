"""CPU: physical-invariant checks of the HalfCheetah physics restatement
(oracle/mjc_oracle.c).  PARITY UNPINNED against MuJoCo itself (absent from this environment and
from the reference tree); these tests pin what can be pinned without it: the compiled model
against the XML, conservation laws, equilibrium, and the env-level reward/obs algebra of
envpool/mujoco/gym/half_cheetah.h:136-177."""
import numpy as np
import pytest

from helpers import HC_OPTIONS, assert_hc_env_algebra, hc_options_id


@pytest.fixture()
def sim():
    from oracle.oracle_lib import MjcSim

    s = MjcSim()
    yield s
    s.close()


def test_compiled_model_matches_xml(sim):
    c = sim.constants()
    assert abs(c["mass"].sum() - 14.0) < 1e-12          # settotalmass="14"
    # inertiafromgeom at uniform density: mass ratios are capsule-volume ratios
    r = 0.046
    vol = lambda h: np.pi * r * r * 2 * h + 4 / 3 * np.pi * r ** 3
    v = np.array([vol(.5) + vol(.15), vol(.145), vol(.15), vol(.094), vol(.133), vol(.106),
                  vol(.07)])
    np.testing.assert_allclose(c["mass"] / 14.0, v / v.sum(), rtol=1e-12)
    assert np.all(c["iyy"] > 0) and np.all(c["dof_invweight0"] > 0)
    # single-capsule bodies: CoM is the geom centre given in the XML
    np.testing.assert_allclose(c["com"][1], [0.1, -0.13], atol=1e-15)
    np.testing.assert_allclose(c["com"][6], [0.045, -0.07], atol=1e-15)


def test_free_fall_and_translation_invariance(sim):
    sim.qpos[:] = 0
    sim.qvel[:] = 0
    sim.qpos[1] = 3.0                                    # far above the floor: no contacts
    sim.step(np.zeros(6))
    assert sim.nefc == 0
    np.testing.assert_allclose(sim.qvel[1], -9.81 * 0.01, rtol=1e-12)
    np.testing.assert_allclose(sim.qvel[[0, 2, 3, 4, 5, 6, 7, 8]], 0, atol=1e-12)
    # shifting x must not change the dynamics
    from oracle.oracle_lib import MjcSim

    a, b = MjcSim(), MjcSim()
    rng = np.random.default_rng(0)
    q0, v0 = rng.uniform(-.1, .1, 9), rng.normal(0, .1, 9)
    a.qpos[:] = q0; a.qvel[:] = v0
    b.qpos[:] = q0; b.qvel[:] = v0; b.qpos[0] += 3.0
    for _ in range(200):
        act = rng.uniform(-1, 1, 6)
        a.step(act); b.step(act)
    np.testing.assert_allclose(b.qpos[0] - 3.0, a.qpos[0], atol=1e-9)
    np.testing.assert_allclose(b.qpos[1:], a.qpos[1:], atol=1e-9)


def test_settles_on_the_floor(sim):
    sim.qpos[:] = 0
    sim.qvel[:] = 0
    for _ in range(1500):
        sim.step(np.zeros(6))
    assert sim.nefc > 0                                   # resting on contacts
    assert np.abs(sim.qvel).max() < 1e-4                  # at rest
    assert -0.3 < sim.qpos[1] < 0.05                      # torso height plausible
    assert np.all(np.isfinite(sim.qpos))


def test_joint_limits_hold(sim):
    sim.qpos[:] = 0
    sim.qvel[:] = 0
    sim.qpos[1] = 3.0
    lo = np.array([-.52, -.785, -.4, -1, -1.2, -.5])
    hi = np.array([1.05, .785, .785, .7, .87, .5])
    for _ in range(300):
        sim.step(np.ones(6))
        sim.qpos[1] = 3.0; sim.qvel[1] = 0                # keep it airborne
    assert np.all(sim.qpos[3:] <= hi + 0.15) and np.all(sim.qpos[3:] >= lo - 0.15)


def test_env_reward_and_obs_algebra():
    from oracle.oracle_lib import OraclePool

    n = 8
    p = OraclePool("HalfCheetah", n, seed=3, max_episode_steps=1000)
    s = p.reset()
    assert s["obs"].shape == (n, 17) and s["obs"].dtype == np.float64
    assert np.abs(s["obs"][:, :8]).max() <= 0.1 + 1e-12   # qpos[1:] = U(-.1,.1)
    assert (s["reward"] == 0).all() and (s["elapsed_step"] == 0).all()
    rng = np.random.default_rng(1)
    x_prev = np.zeros(n)
    first = True
    for t in range(30):
        a = rng.uniform(-1, 1, (n, 6))
        s = p.step(a)
        xv, x = s["info:x_velocity"], s["info:x_position"]
        ctrl = 0.1 * (a * a).sum(1)
        np.testing.assert_allclose(s["info:reward_ctrl"], -ctrl, rtol=1e-12)
        np.testing.assert_array_equal(s["info:reward_run"], xv)
        np.testing.assert_array_equal(s["reward"], (xv - ctrl).astype(np.float32))
        if not first:
            np.testing.assert_allclose(xv, (x - x_prev) / 0.05, rtol=1e-9, atol=1e-12)
        x_prev, first = x.copy(), False
        assert (s["elapsed_step"] == t + 1).all() and not s["done"].any()
    # truncation at max_episode_steps, then auto-reset
    p = OraclePool("HalfCheetah", 2, seed=3, max_episode_steps=5)
    p.reset()
    for t in range(5):
        s = p.step(np.zeros((2, 6)))
    assert s["done"].all() and s["trunc"].all()
    s = p.step(np.zeros((2, 6)))
    assert (s["elapsed_step"] == 0).all() and (s["reward"] == 0).all()


def test_bias_force_satisfies_lagranges_equations(sim):
    """Independent of MuJoCo's conventions: for T = 1/2 v^T M(q) v and V = sum m |g| z the bias
    force of the restatement (computed from body accelerations, RNE style) must equal
    c_i = sum_jk (dM_ij/dq_k - 1/2 dM_jk/dq_i) v_j v_k + dV/dq_i (central differences of the
    restatement's own M and V).  Pins kinematics, Jacobians, inertia and the Coriolis /
    centrifugal / gravity terms against each other; the soft-constraint model is what stays
    unpinned."""
    rng = np.random.default_rng(3)
    eps = 1e-6
    for _ in range(20):
        q = rng.uniform(-0.6, 0.6, size=9)
        v = rng.normal(0, 2.0, size=9)
        M, c, _ = sim.dynamics(q, v)
        np.testing.assert_allclose(M, M.T, rtol=0, atol=1e-12)
        assert np.linalg.eigvalsh(M).min() > 0
        dM = np.zeros((9, 9, 9))      # dM[k] = dM/dq_k
        dV = np.zeros(9)
        for k in range(9):
            dq = np.zeros(9)
            dq[k] = eps
            Mp, _, Vp = sim.dynamics(q + dq, v)
            Mm, _, Vm = sim.dynamics(q - dq, v)
            dM[k] = (Mp - Mm) / (2 * eps)
            dV[k] = (Vp - Vm) / (2 * eps)
        want = np.einsum("kij,j,k->i", dM, v, v) - 0.5 * np.einsum("ijk,j,k->i", dM, v, v) + dV
        np.testing.assert_allclose(c, want, rtol=0, atol=2e-6 * (1 + np.abs(want).max()))
    # the inertia does not depend on the root translation, and momentum rows are plain sums
    M0, _, _ = sim.dynamics(np.zeros(9), np.zeros(9))
    M1, _, _ = sim.dynamics(np.r_[3.0, -1.0, np.zeros(7)], np.zeros(9))
    np.testing.assert_allclose(M0, M1, rtol=0, atol=1e-12)
    total = sim.constants()["mass"].sum()
    assert abs(M0[0, 0] - total) < 1e-12 and abs(M0[1, 1] - total) < 1e-12
    assert abs(M0[0, 1]) < 1e-12


def test_newton_solver_reaches_the_minimiser_of_the_stated_problem(sim):
    """The constraint solve is a convex program: qacc = argmin_a 1/2 (a - a_s)' M (a - a_s) +
    sum_i 1/2 D_i min(0, J_i a - aref_i)^2.  An independent optimiser (scipy, trust-region
    Newton on the exact gradient / Hessian of that cost) started from qacc_smooth must land on the
    restatement's answer, and the answer must satisfy the optimality condition -- which pins
    the hand-written Newton iteration, its line search and its stopping rules (what the CUDA
    kernels restate once more) to the problem they claim to solve.  States: contact-rich
    (folded legs near the floor, fast) with joint limits active."""
    from scipy.optimize import minimize

    rng = np.random.default_rng(11)
    checked = 0
    for trial in range(60):
        sim.qpos[:] = rng.uniform(-0.1, 0.1, 9)
        sim.qpos[1] = rng.uniform(-0.25, 0.2)
        sim.qpos[2] = rng.uniform(-1.5, 1.5)
        sim.qpos[3:] = rng.uniform(-1.3, 1.3, 6)
        sim.qvel[:] = rng.normal(0, 2.0, 9)
        p = sim.solve_problem()
        M, J, D, aref = p["M"], p["J"], p["D"], p["aref"]
        if len(D) == 0:
            continue
        a_s = np.linalg.solve(M, p["qfrc_smooth"])

        def cost(a):
            r = np.minimum(0.0, J @ a - aref)
            da = a - a_s
            return 0.5 * da @ M @ da + 0.5 * np.sum(D * r * r)

        def grad(a):
            r = np.minimum(0.0, J @ a - aref)
            return M @ (a - a_s) + J.T @ (D * r)

        def hess(a):
            act = (J @ a - aref) < 0
            return M + (J[act].T * D[act]) @ J[act]

        a = p["qacc"]
        scale = 1.0 / (np.trace(M) / 9 * 9)   # the solver's own scaling of its tolerances
        g = grad(a)
        assert scale * np.linalg.norm(g) < 1e-6, (trial, len(D), scale * np.linalg.norm(g))
        ref = minimize(cost, a_s, jac=grad, hess=hess, method="trust-exact",
                       options={"gtol": 1e-12, "maxiter": 500})
        assert cost(a) <= ref.fun * (1 + 1e-9) + 1e-9, (trial, cost(a), ref.fun)
        assert np.linalg.norm(a - ref.x) <= 1e-6 * (1 + np.linalg.norm(ref.x)), (
            trial, len(D), np.linalg.norm(a - ref.x))
        checked += 1
    assert checked >= 40, checked


@pytest.mark.parametrize("opts", HC_OPTIONS, ids=hc_options_id)
def test_oracle_runs_the_task_options(opts):
    """OraclePool with HalfCheetah's task options: every step equals MjcSim stepped by hand
    frame_skip times from the same state, bit for bit, and the env-layer algebra holds exactly
    on the oracle's own outputs.  max_episode_steps 12 puts an auto-reset (with this reset noise
    scale) inside the 20 steps."""
    import ctypes

    from oracle.oracle_lib import MjcSim, OraclePool, lib

    n, T = 6, 20
    p = OraclePool("HalfCheetah", n, seed=4, max_episode_steps=12, **opts)
    scale = opts["reset_noise_scale"]
    out = p.reset()
    assert np.abs(out["obs"][:, :8]).max() <= abs(scale)       # qpos[1:] ~ U(-s, s)
    if scale == 0.0:
        assert not out["obs"].view(np.uint64).any()             # +0.0, bit for bit
    else:
        assert np.abs(out["obs"][:, 8:]).max() > abs(scale)     # N(0, s) has tails past |s|
    L = lib()
    L.mjc_warm_mut.restype = ctypes.POINTER(ctypes.c_double)
    L.mjc_warm_mut.argtypes = [ctypes.c_void_p]
    sim = MjcSim()
    warm = np.ctypeslib.as_array(L.mjc_warm_mut(sim.d), shape=(9,))
    rng = np.random.default_rng(2)
    resets = 0
    for t in range(T):
        before = np.array([p.mjc_get(e) for e in range(n)])
        a = rng.uniform(-1.5, 1.5, (n, 6))
        out = p.step(a)
        assert_hc_env_algebra(out, before[:, 0], a, opts, ctx=f"t={t}")
        resets += int((out["elapsed_step"] == 0).sum())
        for e in np.nonzero(out["elapsed_step"] > 0)[0]:
            sim.qpos[:], sim.qvel[:], warm[:] = before[e, :9], before[e, 9:18], before[e, 18:]
            sim.step(a[e], opts["frame_skip"])
            np.testing.assert_array_equal(p.mjc_get(e), np.r_[sim.qpos, sim.qvel, warm])
            np.testing.assert_array_equal(out["obs"][e], np.r_[sim.qpos[1:], sim.qvel])
    assert resets == n


def test_default_options_reproduce_the_recorded_outputs():
    """A HalfCheetah OraclePool left at its default options gives, byte for byte, the outputs the
    oracle gave when the options were still constants: sha256 over every column of two resets
    and 25 steps (a truncation and an auto-reset among them), recorded then."""
    import hashlib

    from oracle.oracle_lib import OraclePool

    p = OraclePool("HalfCheetah", 16, seed=7, max_episode_steps=20)
    rng = np.random.default_rng(21)
    outs = [p.reset(), p.reset()]
    outs += [p.step(rng.uniform(-1.5, 1.5, size=(16, 6))) for _ in range(25)]
    h = hashlib.sha256()
    for o in outs:
        for k in sorted(o):
            h.update(k.encode())
            h.update(np.ascontiguousarray(o[k]).tobytes())
    assert h.hexdigest() == "89f0d446e730be3ba622b28a01f3a3b0cd3c4d7d76fac9799439d60cb97d2f63"
