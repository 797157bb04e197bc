"""GPU: HalfCheetah (two lanes per env) against the CPU restatement of the same
pipeline (oracle/mjc_oracle.c).  PARITY UNPINNED against MuJoCo 3.6.0 itself -- see the
oracle's header and DESIGN.md.  Tolerances: the kernel and the oracle differ only in
summation order / FMA contraction / libm (1e-16 relative per operation); one teacher-forced
env step (5 mj_steps, Newton solves included) must agree to 1e-9; free-running trajectories
are compared over a short horizon because contact dynamics amplify rounding noise (the
reference's own precedent for MuJoCo: 5e-3 over <= 64 steps on arm64,
mujoco_gym_align_test.py:42-43,93-94)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KEYS_EXACT = ("info:env_id", "info:players.env_id", "elapsed_step", "done", "discount",
              "step_type", "trunc")


def _relerr(g, w):
    return np.abs(g - w) / (1 + np.abs(w))


def test_reset_draws_match_oracle_bitwise(capi):
    """Reset = 9 uniform_real + 9 normal_distribution draws (half_cheetah.h:105-116) on the
    device mt19937; qpos noise must be bit-exact, qvel noise within 2 ulp (device log/sqrt)."""
    from oracle.oracle_lib import OraclePool

    n = 512
    pool = capi.CPool("HalfCheetah", n, seed=5, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=5, max_episode_steps=1000)
    g, w = pool.reset(), orc.reset()
    np.testing.assert_array_equal(g["obs"][:, :8], w["obs"][:, :8])
    np.testing.assert_allclose(g["obs"][:, 8:], w["obs"][:, 8:], rtol=1e-14, atol=1e-16)
    for k in KEYS_EXACT + ("reward",):
        np.testing.assert_array_equal(g[k], w[k])
    # a second reset consumes the cached second normal of each pair (saved-state parity)
    g, w = pool.reset(), orc.reset()
    np.testing.assert_allclose(g["obs"], w["obs"], rtol=1e-14, atol=1e-16)


def test_teacher_forced_env_step(capi):
    from oracle.oracle_lib import OraclePool

    n, T = 256, 80
    rng = np.random.default_rng(3)
    pool = capi.CPool("HalfCheetah", n, seed=1, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=1, max_episode_steps=1000)
    pool.reset(), orc.reset()
    worst = 0.0
    for t in range(T):
        st = pool.state_arrays(pool.state_export())
        rs = st["rstate"]                       # SoA [32, n]: qpos 0-8, qvel 9-17, warm 18-26
        for e in range(n):
            orc.mjc_set(e, rs[:27, e], int(st["flags"][e] & 1), int(st["flags"][e] >> 1))
        a = rng.uniform(-1, 1, size=(n, 6))
        g, w = pool.step(a), orc.step(a)
        for k in KEYS_EXACT:
            np.testing.assert_array_equal(g[k], w[k])
        for k in ("obs", "info:x_position", "info:x_velocity", "info:reward_run",
                  "info:reward_ctrl"):
            err = _relerr(g[k], w[k]).max()
            worst = max(worst, err)
            assert err <= 1e-9, (t, k, err)
        assert _relerr(g["reward"], w["reward"]).max() <= 1e-6
    print("teacher-forced worst rel err", worst)


def test_free_running_short_horizon(capi):
    from oracle.oracle_lib import OraclePool

    n, T = 512, 40
    rng = np.random.default_rng(4)
    pool = capi.CPool("HalfCheetah", n, seed=2, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=2, max_episode_steps=1000)
    pool.reset(), orc.reset()
    for t in range(T):
        a = rng.uniform(-1, 1, size=(n, 6))
        g, w = pool.step(a), orc.step(a)
        err = _relerr(g["obs"], w["obs"])
        # median stays at rounding level; the tail is contact-event amplification
        assert np.median(err.max(axis=1)) <= 1e-9, (t, np.median(err.max(axis=1)))
        assert (err.max(axis=1) <= 1e-5).mean() >= 0.99, (t, err.max())


def test_rollout_and_truncation_and_sharding(capi):
    import torch

    n, T = 1000, 12
    rng = np.random.default_rng(5)
    acts = rng.uniform(-1, 1, size=(T, n, 6))
    host = capi.CPool("HalfCheetah", n, seed=9, max_episode_steps=7)
    roll = capi.CPool("HalfCheetah", n, seed=9, max_episode_steps=7)
    lo = capi.CPool("HalfCheetah", n // 2, seed=9, max_episode_steps=7)
    hi = capi.CPool("HalfCheetah", n // 2, seed=9, max_episode_steps=7,
                    env_id_offset=n // 2)
    ref = [host.reset()] + [host.step(acts[t]) for t in range(T)]
    assert ref[7]["trunc"].all() and ref[7]["done"].all()          # max_episode_steps=7
    assert (ref[8]["elapsed_step"] == 0).all()                      # auto-reset next step
    lo.reset(), hi.reset()
    for t in range(T):
        gl, gh = lo.step(acts[t][: n // 2]), hi.step(acts[t][n // 2:])
        for k in ref[t + 1]:
            np.testing.assert_array_equal(np.concatenate([gl[k], gh[k]]), ref[t + 1][k])
    roll.reset_device()
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((T, n) + k.shape, dtype=tdt[k.dtype], device="cuda")
            for k in roll.keys]
    roll.rollout_device(torch.from_numpy(acts).cuda(), T, cols)
    roll.sync()
    for t in range(T):
        for k, c in zip(roll.keys, cols):
            np.testing.assert_array_equal(c[t].cpu().numpy(), ref[t + 1][k.name])


def test_python_api_halfcheetah(capi):
    import envpool_b200 as ep

    env = ep.make_gym("HalfCheetah-v4", num_envs=64, seed=0)
    obs, info = env.reset()
    assert obs.shape == (64, 17) and obs.dtype == np.float64
    a = np.random.default_rng(0).uniform(-1, 1, size=(64, 6))
    obs, rew, term, trunc, info = env.step(a)
    assert rew.dtype == np.float32 and not term.any() and not trunc.any()
    assert set(info) >= {"reward_run", "reward_ctrl", "x_position", "x_velocity"}
    np.testing.assert_allclose(info["reward_ctrl"], -0.1 * (a * a).sum(1), rtol=1e-12)
    assert env.spec.config.max_episode_steps == 1000

