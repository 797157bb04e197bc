"""CPU: Jumanji Game2048-v1 -- the oracle (oracle/g2048_oracle.c) against the fixtures recorded from
the reference's own AsyncEnvPool<Game2048Env> (tests/golden/game2048/), its random-cell recipe
against libstdc++ itself on crafted engine states, and the spec / registry surface of the
pybind module (no GPU needed)."""
import glob
import json
import os

import numpy as np
import pytest

from helpers import GOLDEN, assert_batch_equal
from test_oracle_rng_vs_libstdcxx import untemper

G2048 = os.path.join(GOLDEN, "game2048")
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(G2048, "*.npz")))


def load_fixture(name):
    z = np.load(os.path.join(G2048, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    return meta, {k: z[k] for k in z.files if k != "meta"}


def cells(text, n):
    """A board string as the reference parses it: comma-separated, missing cells 0."""
    if not text:
        return None
    v = [int(t) for t in text.split(",")][:n]
    return np.array(v + [0] * (n - len(v)), dtype=np.int32)


def oracle_for(meta, **over):
    from oracle.g2048_lib import Game2048Oracle

    m = dict(meta, **over)
    return Game2048Oracle(m["num_envs"], seed=m["seed"], max_episode_steps=m["max_episode_steps"],
                          add_random_cell=m["add_random_cell"],
                          initial=cells(m["initial_board"], 16),
                          replay=cells(m["replay_boards"], 512))


def test_fixtures_cover_the_issue_cases():
    assert FIXTURES == ["dead_initial_board", "default", "max_steps_1", "max_steps_5",
                        "no_random_cell", "short_replay"]
    meta, gold = load_fixture("default")
    assert meta["num_envs"] == 64 and gold["actions"].shape == (1000, 64)
    assert set(np.unique(gold["actions"])) >= {-5, 4, -2**31, 2**31 - 1, 0, 1, 2, 3}
    meta, gold = load_fixture("dead_initial_board")
    assert gold["done"].all() and (gold["step_type"] == 0).all()   # every row is a reset
    meta, gold = load_fixture("max_steps_5")
    assert gold["trunc"].any() and (gold["trunc"] <= gold["done"]).all()


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_fixture(name):
    meta, gold = load_fixture(name)
    orc = oracle_for(meta)
    keys = [k for k in gold if k != "actions"]
    assert_batch_equal(orc.reset(), {k: gold[k][0] for k in keys}, "Game2048", 0.0,
                       f"{name} reset")
    for t, a in enumerate(gold["actions"]):
        assert_batch_equal(orc.step(a), {k: gold[k][t + 1] for k in keys}, "Game2048", 0.0,
                           f"{name} t={t}")


def test_seeded_reset_known_answer():
    """seed 7, 4 envs: (cell, exponent) of each reset board's one tile, printed by the compiled
    reference.  Drawing the position before the value would give (1, 1), (13, 1), (0, 1),
    (12, 2)."""
    from oracle.g2048_lib import Game2048Oracle

    b = Game2048Oracle(4, seed=7).reset()["obs:board"]
    got = [(int(np.flatnonzero(x)[0]), int(x.ravel()[np.flatnonzero(x)[0]])) for x in b]
    assert got == [(12, 1), (15, 2), (8, 1), (0, 1)]
    assert all(np.count_nonzero(x) == 1 for x in b)


def _move_line(line):
    """Independent statement of a line slide: drop gaps, merge equal neighbours once, from
    the edge the tiles slide to."""
    tiles = [int(v) for v in line if v]
    out, reward, i = [], 0.0, 0
    while i < len(tiles):
        if i + 1 < len(tiles) and tiles[i] == tiles[i + 1]:
            out.append(tiles[i] + 1)
            reward += 2.0 ** (tiles[i] + 1)
            i += 2
        else:
            out.append(tiles[i])
            i += 1
    return out + [0] * (4 - len(out)), reward


def rule_move(board, action):
    """One move of a 4x4 board (0 up, 1 right, 2 down, 3 left) and its reward."""
    b = np.array(board, dtype=np.int32)
    view = {0: lambda x: x.T, 1: lambda x: x[:, ::-1], 2: lambda x: x[::-1, :].T,
            3: lambda x: x}[action]
    out = b.copy()
    reward = 0.0
    src, dst = view(b), view(out)
    for i in range(4):
        line, r = _move_line(src[i])
        dst[i] = line
        reward += r
    return out, reward


def rule_mask(board):
    return np.array([not np.array_equal(rule_move(board, a)[0], board) for a in range(4)])


# the reference test's fixed rollout: this board, add_random_cell=False, six moves
RULE_BOARD = np.array([[1, 1, 2, 2], [3, 4, 0, 0], [0, 2, 0, 0], [0, 5, 0, 0]], dtype=np.int32)
RULE_ACTIONS = [3, 0, 1, 2, 3, 0]


def test_oracle_fixed_rollout_matches_the_rules():
    from oracle.g2048_lib import Game2048Oracle

    orc = Game2048Oracle(1, seed=0, add_random_cell=False, initial=RULE_BOARD.ravel())
    board = RULE_BOARD.copy()
    out = orc.reset()
    np.testing.assert_array_equal(out["obs:board"][0], board)
    np.testing.assert_array_equal(out["obs:action_mask"][0], rule_mask(board))
    assert out["info:highest_tile"][0] == 32
    for a in RULE_ACTIONS:
        board, reward = rule_move(board, a)
        out = orc.step(np.array([a], np.int32))
        np.testing.assert_array_equal(out["obs:board"][0], board)
        np.testing.assert_array_equal(out["obs:action_mask"][0], rule_mask(board))
        assert float(out["reward"][0]) == reward
        assert bool(out["done"][0]) == (not rule_mask(board).any())
        assert not out["trunc"][0]
        assert out["info:highest_tile"][0] == 2 ** board.max()


def test_reward_is_summed_in_line_order():
    """Float rewards: line totals are added for lines 0..3.  With a 2^27 merge in line 0 and
    three 2^2 merges after it, every later 4 is lost to rounding (half an ulp of 2^27 is 8);
    summing the other way round keeps 12 of them and rounds up to 2^27 + 16."""
    from oracle import g2048_lib

    board = np.zeros((4, 4), np.int32)
    board[0, :2] = 26        # row 0 moving left: one merge -> 2^27
    board[1:, :2] = 1        # rows 1..3: one merge each -> 2^2
    orc = g2048_lib.Game2048Oracle(1, seed=0, add_random_cell=False, initial=board.ravel())
    orc.reset()
    r = orc.step(np.array([3], np.int32))["reward"][0]
    f = np.float32
    assert r == f(2.0**27)
    assert ((f(4) + f(4)) + f(4)) + f(2.0**27) == f(2.0**27 + 16)
    if g2048_lib.ref_available():
        ref = g2048_lib.Game2048Ref(1, seed=0, add_random_cell=False,
                                    initial_board=",".join(map(str, board.ravel())))
        ref.reset()
        assert ref.step(np.array([3], np.int32))["reward"][0] == r


def crafted_state(outputs, idx=100, seed=3):
    """A seeded engine state whose next len(outputs) draws are `outputs` (None = leave)."""
    mt = np.zeros(624, np.uint32)
    s = seed
    for i in range(624):
        mt[i] = s
        s = (1812433253 * (s ^ (s >> 30)) + i + 1) & 0xFFFFFFFF
    for k, o in enumerate(outputs):
        if o is not None:
            mt[idx + k] = untemper(o)
    return mt, idx


# canonical = (w0 + w1 * 2^32) / 2^64: w1 decides whether it lies below 0.1
P01 = int(0.1 * 2**32)
CASES = {
    "plain, 16 empty": ([None, None, None], 16),
    "value 2 (canonical just below 0.1)": ([0xFFFFFFFF, P01 - 1, None], 11),
    "value 1 (canonical just above 0.1)": ([0, P01 + 1, None], 11),
    "Lemire rejection (word 0, 3 empty)": ([None, None, 0, None], 3),
    "two Lemire rejections (7 empty)": ([None, None, 0, 0, 123456789], 7),
    "one empty cell still draws a word": ([None, None, 77, 5], 1),
    "no rejection for a power of two (word 0, 8 empty)": ([None, None, 0, 99], 8),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_random_cell_recipe_equals_libstdcxx(case):
    """Value (bernoulli(0.1): generate_canonical<double>, 2 words) before position
    (uniform_int(0, n-1): Lemire, 1 word plus rejections), on crafted engine states; then both
    engines must stand at the same word."""
    from oracle.g2048_lib import Game2048Oracle, StdRng

    outputs, n = CASES[case]
    mt, idx = crafted_state(outputs)
    std = StdRng()
    std.set(mt, idx)
    orc = Game2048Oracle(1, seed=0)
    orc.set_rng(0, mt, idx)
    want = std.random_cell(n)
    assert orc.random_cell(0, n) == want
    assert orc.draw(0) == std.next()
    if "value 2" in case:
        assert want[0] == 2
    if "value 1" in case:
        assert want[0] == 1


def test_bernoulli_equals_libstdcxx_on_seeded_streams():
    """Seeded engine states (read position 624: the next draw regenerates the table) load
    into both engines identically, and bernoulli_distribution agrees draw by draw."""
    from oracle.g2048_lib import Game2048Oracle, StdRng

    std = StdRng()
    for seed in (0, 7, 12345):
        mt, _ = crafted_state([], seed=seed)
        std.set(mt, 624)
        orc = Game2048Oracle(1, seed=0)
        orc.set_rng(0, mt, 624)
        assert [orc.draw(0) for _ in range(700)] == [std.next() for _ in range(700)]
        for p in (0.1, 0.5, 0.0, 1.0):
            got = [orc.bernoulli(0, p) for _ in range(200)]
            want = [std.bernoulli(p) for _ in range(200)]
            assert got == want, (seed, p)


# ---------------------------------------------------------------- spec and registry ------
def test_spec_keys_defaults_and_alias(engine_built):
    import envpool_b200 as ep
    from envpool_b200.jumanji import jumanji_envpool as jm

    S = jm._Game2048EnvSpec
    assert S._config_keys[10:] == ["game2048_initial_board", "game2048_replay_boards",
                                   "game2048_add_random_cell"]
    assert S._default_config_values[10:] == ("", "", True)
    assert list(S._state_keys) == ["info:env_id", "info:players.env_id", "elapsed_step", "done",
                                   "reward", "discount", "step_type", "trunc", "obs:board",
                                   "obs:action_mask", "info:highest_tile"]
    assert list(S._action_keys) == ["env_id", "players.env_id", "action"]
    ids = ep.list_all_envs()
    assert "Game2048-v1" in ids and "Jumanji/Game2048-v1" in ids
    for tid in ("Game2048-v1", "Jumanji/Game2048-v1"):
        spec = ep.make_spec(tid, num_envs=3)
        assert spec.config.max_episode_steps == 1000
        assert spec.config.game2048_add_random_cell is True
        st = dict(zip(spec._state_keys, spec._state_spec))
        assert st["obs:board"][1] == [4, 4] and np.dtype(st["obs:board"][0]) == np.int32
        assert st["obs:action_mask"][1] == [4] and np.dtype(st["obs:action_mask"][0]) == np.bool_
        assert st["obs:action_mask"][2] == (False, True)
        assert st["info:highest_tile"][1] == [] and st["info:highest_tile"][2] == (1, 2**30)
        act = dict(zip(spec._action_keys, spec._action_spec))["action"]
        assert act[1] == [-1] and act[2] == (0, 3)


def test_observation_space_is_a_dict_and_dm_spec_a_namedtuple(engine_built):
    import envpool_b200 as ep

    spec = ep.make_spec("Game2048-v1", num_envs=2)
    space = spec.observation_space
    assert isinstance(space, dict) and hasattr(space, "spaces")
    assert list(space.keys()) == ["board", "action_mask"]
    assert space["board"].shape == (4, 4) and space["board"].dtype == np.int32
    assert space["action_mask"].shape == (4,)
    assert type(space["action_mask"]).__name__ == "MultiBinary"
    assert spec.action_space.n == 4
    dm = spec.observation_spec()
    assert list(dm._fields) == ["env_id", "players", "board", "action_mask", "highest_tile"]
    # the single-key envs keep their space unchanged
    assert not isinstance(ep.make_spec("CartPole-v1").observation_space, dict)


@pytest.mark.parametrize("kw", [
    dict(game2048_initial_board="1,2,27"),
    dict(game2048_initial_board="-1"),
    dict(game2048_replay_boards=",".join(["0"] * 100 + ["30"])),
    dict(game2048_initial_board="1,x,2"),
    dict(game2048_replay_boards="1,,2"),
])
def test_out_of_range_or_malformed_boards_raise_value_error(engine_built, kw):
    import envpool_b200 as ep

    with pytest.raises(ValueError):
        ep.make_spec("Game2048-v1", num_envs=2, **kw)


def test_boards_in_range_are_accepted(engine_built):
    import envpool_b200 as ep

    ep.make_spec("Game2048-v1", num_envs=2, game2048_initial_board="26,0,1",
                 game2048_replay_boards=",".join(["26"] * 600))
