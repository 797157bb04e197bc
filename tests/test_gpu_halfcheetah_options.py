"""GPU: HalfCheetah's task options (frame_skip, forward_reward_weight, ctrl_cost_weight,
reset_noise_scale) held to the CPU restatement of the pipeline (oracle/mjc_oracle.c), which runs
them as the reference does (half_cheetah.h:84-160), and to the env-layer algebra bit for bit.

The options travel make() / CPool / ShardedPool -> epb_config -> HcParams (csrc/mujoco.cu
hc_setup).  In epb_config a NaN double means "the reference default"; every other value, negative
or -0.0 included, is used as given.  The configurations are the table in helpers.py.

Bars (those of test_gpu_halfcheetah.py): integer and bool columns exact; reset qpos bit-exact and
qvel within rtol 1e-14 (device log / sqrt in the normal draws); float64 columns within 1e-9
relative-absolute per teacher-forced env step; the float32 reward within 1e-6.  Entry points that
issue the same launches agree bit for bit."""
import numpy as np
import pytest

from helpers import HC_DEFAULT, HC_OPTIONS, assert_hc_env_algebra, hc_options_id

pytestmark = pytest.mark.gpu

EXACT = ("info:env_id", "info:players.env_id", "elapsed_step", "done", "discount", "step_type",
         "trunc")
FLOATS = ("obs", "info:reward_run", "info:reward_ctrl", "info:x_position", "info:x_velocity")
INFO = ("reward_run", "reward_ctrl", "x_position", "x_velocity")
# a configuration with every option away from its default and of the "wrong" sign where it has
# one: the cheetah is rewarded for running backwards, its ctrl cost is a bonus, frame_skip 2
ODD = dict(frame_skip=2, forward_reward_weight=-1.0, ctrl_cost_weight=-0.05, reset_noise_scale=1.0)
assert ODD in HC_OPTIONS


def _relerr(g, w):
    g, w = g.astype(np.float64), w.astype(np.float64)
    return np.abs(g - w) / (1 + np.abs(w))


def _same_bytes(got, want, ctx):
    assert set(got) == set(want), ctx
    for k in want:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.dtype == w.dtype and g.shape == w.shape, (ctx, k, g.dtype, w.dtype)
        assert g.tobytes() == w.tobytes(), (ctx, k)


@pytest.mark.parametrize("opts", HC_OPTIONS, ids=hc_options_id)
def test_reset_matches_oracle(capi, opts):
    """Two consecutive resets (the second takes the cached second normal of each pair) against
    the oracle: qpos bit-exact (in the state, so qpos[0] too), qvel to rounding, every other
    column exact.  At scale 0 the reset state is +0.0 everywhere and the draws still happen:
    mt_idx equals a default-scale pool's."""
    from oracle.oracle_lib import OraclePool

    n = 512
    pool = capi.CPool("HalfCheetah", n, seed=5, max_episode_steps=1000, **opts)
    orc = OraclePool("HalfCheetah", n, seed=5, max_episode_steps=1000, **opts)
    dflt = capi.CPool("HalfCheetah", n, seed=5, max_episode_steps=1000)
    scale = opts["reset_noise_scale"]
    for r in range(2):
        g, w, d = pool.reset(), orc.reset(), dflt.reset()
        rs = pool.state_arrays(pool.state_export())["rstate"]
        want = np.array([orc.mjc_get(e) for e in range(n)])
        assert rs[:9].T.tobytes() == want[:, :9].tobytes(), (r, "qpos")
        np.testing.assert_allclose(rs[9:18].T, want[:, 9:18], rtol=1e-14, atol=1e-16)
        np.testing.assert_array_equal(g["obs"][:, :8], w["obs"][:, :8])
        np.testing.assert_allclose(g["obs"][:, 8:], w["obs"][:, 8:], rtol=1e-14, atol=1e-16)
        for k in g:
            if k != "obs":
                assert g[k].tobytes() == w[k].tobytes(), (r, k)
        assert np.abs(g["obs"][:, :8]).max() <= abs(scale)
        if scale == 0.0:   # +0.0, not -0.0
            for x in (g["obs"], rs[:18]):
                assert (x == 0).all() and not np.signbit(x).any(), r
            got_idx = pool.state_arrays(pool.state_export())["mt_idx"]
            dflt_idx = dflt.state_arrays(dflt.state_export())["mt_idx"]
            np.testing.assert_array_equal(got_idx, dflt_idx)
        elif scale != HC_DEFAULT["reset_noise_scale"]:
            assert not np.array_equal(g["obs"], d["obs"]), r


@pytest.mark.parametrize("opts", HC_OPTIONS, ids=hc_options_id)
def test_teacher_forced_steps_match_oracle(capi, opts):
    """256 envs, 30 steps, actions uniform in [-1.5, 1.5]: the ctrl cost sees them raw, the
    dynamics clamped.  Before each step the oracle takes the engine's state.  max_episode_steps 12
    puts two auto-resets (drawn with this noise scale) among the steps.  The env-layer algebra is
    checked bit for bit on the full batch of every step."""
    from oracle.oracle_lib import OraclePool

    n, T = 256, 30
    rng = np.random.default_rng(3)
    pool = capi.CPool("HalfCheetah", n, seed=1, max_episode_steps=12, **opts)
    orc = OraclePool("HalfCheetah", n, seed=1, max_episode_steps=12, **opts)
    pool.reset(), orc.reset()
    worst, resets = 0.0, 0
    for t in range(T):
        st = pool.state_arrays(pool.state_export())
        rs, fl = st["rstate"], st["flags"]
        for e in range(n):
            orc.mjc_set(e, rs[:27, e], int(fl[e] & 1), int(fl[e] >> 1))
        a = rng.uniform(-1.5, 1.5, size=(n, 6))
        g, w = pool.step(a), orc.step(a)
        for k in EXACT:
            np.testing.assert_array_equal(g[k], w[k], err_msg=f"t={t} {k}")
        for k in FLOATS:
            err = float(_relerr(g[k], w[k]).max())
            worst = max(worst, err)
            assert err <= 1e-9, (t, k, err)
        assert _relerr(g["reward"], w["reward"]).max() <= 1e-6, t
        assert_hc_env_algebra(g, rs[0], a, opts, ctx=f"t={t}")
        resets += int((g["elapsed_step"] == 0).sum())
    assert resets == 2 * n
    print(f"{hc_options_id(opts)}: worst teacher-forced rel err {worst:.3e}")


def test_every_entry_point_sees_the_pool_options(capi):
    """One state blob, K steps through step, step_device, step_many_device (graph and direct),
    step_many_timed and rollout_device of pools created with ODD: the same launches, so the same
    bits, and the host path obeys the env-layer algebra of ODD.  1000 envs leave the last CTA
    partial; max_episode_steps 5 puts resets with ODD's noise scale inside every chain."""
    import torch

    n, K = 1000, 12
    names = ("step", "step_device", "graph", "direct", "timed", "rollout")
    pools = {k: capi.CPool("HalfCheetah", n, seed=11, max_episode_steps=5, **ODD) for k in names}
    pools["step"].reset()
    blob = pools["step"].state_export()
    for p in pools.values():
        p.state_import(blob)
    rng = np.random.default_rng(n)
    acts = rng.uniform(-1.5, 1.5, size=(K, n, 6))
    d_acts = torch.from_numpy(acts).cuda()
    host = []
    for t in range(K):
        x_before = pools["step"].state_arrays(pools["step"].state_export())["rstate"][0]
        host.append(pools["step"].step(acts[t]))
        assert_hc_env_algebra(host[-1], x_before, acts[t], ODD, ctx=f"host t={t}")
    assert (np.array([h["elapsed_step"] for h in host]) == 0).sum() == 2 * n

    def outputs(p):
        p.sync()
        return {k: v.cpu().numpy() for k, v in p.outputs_torch().items()}

    for t in range(K):
        pools["step_device"].step_device(d_acts[t])
        _same_bytes(outputs(pools["step_device"]), host[t], f"step_device t={t}")
    pools["graph"].step_many_device(d_acts, 0, K, use_graph=True)
    pools["direct"].step_many_device(d_acts, 0, K, use_graph=False)
    assert pools["timed"].step_many_timed(d_acts, 0, K, 4, K) > 0
    p = pools["rollout"]
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((K, n) + k.shape, dtype=tdt[k.dtype], device="cuda") for k in p.keys]
    p.rollout_device(d_acts, K, cols)
    p.sync()
    for t in range(K):
        _same_bytes({k.name: c[t].cpu().numpy() for k, c in zip(p.keys, cols)}, host[t],
                    f"rollout_device t={t}")
    for name in ("graph", "direct", "timed"):
        _same_bytes(outputs(pools[name]), host[-1], f"{name} t={K - 1}")
    want = pools["step"].state_export().tobytes()
    for name in names[1:]:
        assert pools[name].state_export().tobytes() == want, name


def _public_columns(ret, dm):
    """The float columns of a step's return value, by state key."""
    if dm:
        o = ret.observation
        out = {"obs": o.obs, "reward": ret.reward}
        out.update({f"info:{k}": getattr(o, k) for k in INFO})
        return out
    obs, rew, term, trunc, info = ret
    out = {"obs": obs, "reward": rew}
    out.update({f"info:{k}": info[k] for k in INFO})
    return out


@pytest.mark.parametrize("task", ["HalfCheetah-v3", "HalfCheetah-v4", "HalfCheetah-v5"])
def test_make_carries_the_options(capi, task):
    """make_gym / make_gymnasium / make_dm with the options as kwargs equal a CPool with the same
    options bit for bit (outputs and state); without kwargs they equal a CPool left at its
    defaults.  A CPool left at its defaults (NaN in epb_config) equals one given 5, 0.1, 1.0, 0.1
    explicitly."""
    import warnings

    import envpool_b200 as ep

    n, T = 64, 6
    rng = np.random.default_rng(7)
    acts = rng.uniform(-1.5, 1.5, size=(T, n, 6))
    ref = {}
    for name, kw in (("odd", ODD), ("default", {}), ("explicit", HC_DEFAULT)):
        p = capi.CPool("HalfCheetah", n, seed=3, max_episode_steps=1000, **kw)
        outs = [p.reset()] + [p.step(a) for a in acts]
        ref[name] = (outs, p.state_export().tobytes())
    assert ref["default"][1] == ref["explicit"][1]
    for a, b in zip(ref["default"][0], ref["explicit"][0]):
        _same_bytes(a, b, "NaN defaults vs explicit defaults")
    for make, dm in ((ep.make_gym, False), (ep.make_gymnasium, False), (ep.make_dm, True)):
        for name, kw in (("odd", ODD), ("default", {})):
            outs, state = ref[name]
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                env = make(task, num_envs=n, seed=3, **kw)
            r = env.reset()
            obs0 = r.observation.obs if dm else r[0]
            assert obs0.tobytes() == outs[0]["obs"].tobytes(), (make.__name__, name)
            for t in range(T):
                got = _public_columns(env.step(acts[t]), dm)
                _same_bytes(got, {k: outs[t + 1][k] for k in got}, f"{make.__name__} {name} {t}")
            assert env.device_pool.state_export().tobytes() == state, (make.__name__, name)


def test_sharded_pool_carries_the_options(capi):
    """A single-process ShardedPool forwards HalfCheetah's options to its pool; registry defaults
    that change no column (v5's post_constraint and gymnasium_v5_render_camera) keep working,
    passed explicitly too."""
    import torch

    from envpool_b200.sharded import ShardedPool

    n, T = 256, 6
    rng = np.random.default_rng(9)
    acts = rng.uniform(-1.5, 1.5, size=(T, n, 6))
    for task, kw in (("HalfCheetah-v4", dict(forward_reward_weight=-1.0, frame_skip=2)),
                     ("HalfCheetah-v5", dict(post_constraint=True, ctrl_cost_weight=-0.05,
                                             reset_noise_scale=1.0))):
        sp = ShardedPool(task, n, seed=4, **kw)
        opts = {k: v for k, v in kw.items() if k != "post_constraint"}
        ref = capi.CPool("HalfCheetah", n, seed=4, max_episode_steps=1000, **opts)
        out = sp.reset_device()
        sp.pool.sync()
        _same_bytes({k: v.cpu().numpy() for k, v in out.items()}, ref.reset(), f"{task} reset")
        for t in range(T):
            out = sp.step_device(torch.from_numpy(acts[t]).cuda())
            sp.pool.sync()
            _same_bytes({k: v.cpu().numpy() for k, v in out.items()}, ref.step(acts[t]),
                        f"{task} t={t}")
        assert sp.pool.state_export().tobytes() == ref.state_export().tobytes(), task
