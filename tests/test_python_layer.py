"""CPU: host-side Python layer without touching the GPU -- registry contents, spec
tuples / key lists exported by the pybind modules (pinned like
envpool/dummy/dummy_py_envpool_test.py:59-101), tree conversion helpers."""
import numpy as np
import pytest


def test_registry_lists_reference_task_ids(engine_built):
    import envpool_b200 as ep

    ids = ep.list_all_envs()
    for t in ["CartPole-v0", "CartPole-v1", "Pendulum-v0", "Pendulum-v1", "MountainCar-v0",
              "MountainCarContinuous-v0", "Acrobot-v1", "Catch-v0", "FrozenLake-v1",
              "FrozenLake8x8-v1", "Taxi-v3", "NChain-v0", "CliffWalking-v0",
              "CliffWalking-v1", "CliffWalkingSlippery-v1", "Blackjack-v1",
              "HalfCheetah-v3", "HalfCheetah-v4", "HalfCheetah-v5", "phys2d/CartPole-v1",
              "tabular/Blackjack-v0"]:
        assert t in ids


def test_spec_export_format_and_defaults(engine_built):
    import envpool_b200 as ep
    from envpool_b200.classic_control import classic_control_envpool as cc

    S = cc._CartPoleEnvSpec
    assert S._config_keys == ["num_envs", "batch_size", "num_threads", "max_num_players",
                              "thread_affinity_offset", "base_path", "seed", "env_seed",
                              "gym_reset_return_info", "max_episode_steps",
                              "reward_threshold"]
    assert S._default_config_values == (1, 0, 0, 1, -1, "envpool", 42, [], True,
                                        2**31 - 1, 195.0)
    assert S._state_keys == ["info:env_id", "info:players.env_id", "elapsed_step", "done",
                             "reward", "discount", "step_type", "trunc", "obs"]
    assert S._action_keys == ["env_id", "players.env_id", "action"]
    spec = ep.make_spec("CartPole-v1", num_envs=8)
    assert spec.config.batch_size == 8            # 0 -> num_envs (env_spec.h:81-83)
    assert spec.config.max_episode_steps == 500 and spec.reward_threshold == 475.0
    dtype, shape, bounds, ebounds, disc = spec._state_spec[-1]
    assert dtype == np.float32 and shape == [4] and len(ebounds[0]) == 4
    assert spec._action_spec[-1][:3] == (np.dtype(np.int32), [-1], (0, 1))
    with pytest.raises(ValueError):
        ep.make_spec("CartPole-v1", num_envs=2, batch_size=3) if False else \
            S((2, 3, 0, 1, -1, "envpool", 42, [], True, 500, 475.0))
    hc = ep.make_spec("HalfCheetah-v4", num_envs=2)
    assert hc.config.post_constraint is False and hc.config.frame_skip == 5
    assert hc.observation_space.shape == (17,) and hc.action_space.shape == (6,)
    assert hc._state_keys[8:] == ["obs", "info:reward_run", "info:reward_ctrl",
                                  "info:x_position", "info:x_velocity"]
    fl = ep.make_spec("FrozenLake8x8-v1")
    assert fl.observation_space.n == 64 and fl.config.max_episode_steps == 200


def test_seed_list_becomes_env_seed(engine_built):
    import envpool_b200 as ep

    spec = ep.make_spec("CartPole-v1", num_envs=3, seed=[7, 8, 9])
    assert spec.config.env_seed == [7, 8, 9] and spec.config.seed == 0
    with pytest.raises(AssertionError):
        ep.make_spec("CartPole-v1", num_envs=3, seed=[1, 2])


def test_tree_helpers():
    from envpool_b200.python.data import dm_structure, fill_tree, gym_structure, to_namedtuple

    keys = ["info:env_id", "info:players.env_id", "elapsed_step", "done", "reward",
            "discount", "step_type", "trunc", "obs", "info:state"]
    vals = list(range(len(keys)))
    g = fill_tree(gym_structure(keys), vals)
    assert g["info"] == {"env_id": 0, "players": {"env_id": 1}, "state": 9}
    assert g["obs"] == 8 and g["trunc"] == 7
    d = to_namedtuple("State", fill_tree(dm_structure("State", keys), vals))
    assert d.State.obs == 8 and d.State.players.env_id == 1 and d.State.state == 9
    assert d.step_type == 6


def test_adapter_folds_without_a_device(engine_built):
    """The dm / gymnasium adapters fold the flat `_recv()` column list (state-key order)
    into TimeStep / the gymnasium 5-tuple; the fold needs no engine instance."""
    from envpool_b200.classic_control import CartPoleDMEnvPool, CartPoleGymnasiumEnvPool

    assert CartPoleGymnasiumEnvPool._state_keys == [
        "info:env_id", "info:players.env_id", "elapsed_step", "done", "reward", "discount",
        "step_type", "trunc", "obs"]
    n = 3
    ids = np.arange(n, dtype=np.int32)
    done, trunc = np.array([0, 1, 1], bool), np.array([0, 0, 1], bool)
    obs = np.arange(4 * n, dtype=np.float32).reshape(n, 4)
    cols = [ids, ids, np.full(n, 7, np.int32), done, np.ones(n, np.float32),
            (~done).astype(np.float32), np.array([1, 2, 2], np.int32), trunc, obs]
    o, info = CartPoleGymnasiumEnvPool._to(None, cols, True, True)
    assert o is obs and info["env_id"] is ids and info["players"]["env_id"] is ids
    assert (info["elapsed_step"] == 7).all()
    o, rew, term, tr, info = CartPoleGymnasiumEnvPool._to(None, cols, False, True)
    assert term.tolist() == [False, True, False] and tr.tolist() == [False, False, True]
    ts = CartPoleDMEnvPool._to(None, cols, False, True)
    assert ts.observation.obs is obs and ts.observation.players.env_id is ids
    assert ts.last().tolist() == [False, True, True] and ts.mid().tolist() == [True, False, False]
    with pytest.raises(RuntimeError):
        CartPoleDMEnvPool.xla(None)


def test_halfcheetah_refuses_frame_skip_below_one(engine_built):
    """The reference takes frame_skip substeps and divides by dt = frame_skip * timestep
    (half_cheetah.h:151-152): 0 gives a NaN reward, so the pool refuses it (and anything below)
    before it touches a device."""
    import warnings

    import envpool_b200 as ep

    for make in (ep.make_gym, ep.make_gymnasium, ep.make_dm):
        for fs in (0, -1):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                with pytest.raises(ValueError, match="frame_skip"):
                    make("HalfCheetah-v4", num_envs=2, frame_skip=fs)
