"""CPU: Jumanji Minesweeper-v0 -- the oracle (oracle/ms_oracle.c) against the fixtures recorded from
the reference's own AsyncEnvPool<MinesweeperEnv> (tests/golden/minesweeper/), the mine placement
(the oracle's full shuffle and a model of the kernel's register-only one) against libstdc++'s
std::shuffle on crafted engine states, Reveal on hand-built boards, and the spec / registry
surface of the pybind module (no GPU needed)."""
import glob
import json
import os

import numpy as np
import pytest

from helpers import GOLDEN, assert_batch_equal
from test_game2048 import crafted_state

MS = os.path.join(GOLDEN, "minesweeper")
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MS, "*.npz")))
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1


def load_fixture(name):
    z = np.load(os.path.join(MS, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    return meta, {k: z[k] for k in z.files if k != "meta"}


def parse_config(meta):
    """The four config strings of a fixture as the reference reads them (the fixtures use plain
    integers and exactly representable floats): (mines100 | None, replay | None, rewards, done)."""
    mines = None
    locs = [int(t) for t in meta["mine_locations"].split(",")] if meta["mine_locations"] else []
    locs = [v for v in locs if 0 <= v < 100]
    if locs:
        mines = np.zeros(100, np.int32)
        mines[locs] = 1
    replay = rewards = done = None
    if meta["replay_boards"]:
        v = [int(t) for t in meta["replay_boards"].split(",")][:3200]
        replay = np.array(v + [-1] * (3200 - len(v)), np.int32)
        r = [float(t) for t in meta["replay_rewards"].split(",")][:32] if meta[
            "replay_rewards"] else []
        rewards = np.array(r + [0.0] * (32 - len(r)), np.float32)
        d = [t in ("1", "True", "true") for t in meta["replay_done"].split(",")][:32] if meta[
            "replay_done"] else []
        done = np.array(d + [False] * (32 - len(d)), np.uint8)
    return mines, replay, rewards, done


def oracle_for(meta, **over):
    from oracle.ms_lib import MinesweeperOracle

    m = dict(meta, **over)
    mines, replay, rewards, done = parse_config(m)
    return MinesweeperOracle(m["num_envs"], seed=m["seed"],
                             max_episode_steps=m["max_episode_steps"], mines=mines,
                             replay=replay, rewards=rewards, done=done)


def test_fixtures_cover_the_issue_cases():
    assert FIXTURES == ["configured_mines", "default", "max_steps_1", "max_steps_5",
                        "mines_out_of_range", "replay_done", "short_replay"]
    meta, gold = load_fixture("default")
    assert meta["num_envs"] == 64 and gold["actions"].shape == (200, 64, 2)
    assert set(np.unique(gold["actions"])) >= {-5, 10, INT32_MIN, INT32_MAX} | set(range(10))
    assert (gold["obs:num_mines"] == 10).all()
    _, gold = load_fixture("configured_mines")
    assert (gold["obs:num_mines"] == 5).all()            # duplicates and -3, 100, 250 dropped
    _, gold = load_fixture("mines_out_of_range")
    assert (gold["obs:num_mines"] == 10).all()           # random placement
    _, gold = load_fixture("short_replay")
    assert gold["obs:step_count"].max() > 32             # the env plays on after the replay
    _, gold = load_fixture("replay_done")
    assert gold["done"][1:].any() and gold["obs:step_count"].max() == 2
    _, gold = load_fixture("max_steps_5")
    assert gold["trunc"].any() and (gold["trunc"] <= gold["done"]).all()


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_reference_fixture(name):
    meta, gold = load_fixture(name)
    orc = oracle_for(meta)
    keys = [k for k in gold if k != "actions"]
    assert_batch_equal(orc.reset(), {k: gold[k][0] for k in keys}, "Minesweeper", 0.0,
                       f"{name} reset")
    for t, a in enumerate(gold["actions"]):
        assert_batch_equal(orc.step(a), {k: gold[k][t + 1] for k in keys}, "Minesweeper", 0.0,
                           f"{name} t={t}")


SEED7_MINES = [22, 27, 32, 45, 51, 52, 55, 76, 87, 93]


def test_seeded_mines_known_answer():
    """std::mt19937(7) -- env 0 of a seed-7 pool -- places mines on these cells (computed with
    libstdc++ directly); the oracle's shuffle and, when the build made it, the reference's own
    env agree: a click on each of them hits a mine, a click anywhere else does not."""
    from oracle import ms_lib

    orc = ms_lib.MinesweeperOracle(1, seed=7)
    assert sorted(orc.shuffle(0)[:10]) == SEED7_MINES
    std = ms_lib.StdShuffle()
    mt, _ = crafted_state([], seed=7)
    std.set(mt, 624)
    assert sorted(std.shuffle()[:10]) == SEED7_MINES
    if ms_lib.ref_available():
        # env e of a pool is seeded 7 + e: one single-env pool per clicked cell
        hits = []
        for cell in range(100):
            one = ms_lib.MinesweeperRef(1, seed=7, num_threads=1)
            one.reset()
            out = one.step(np.array([[cell // 10, cell % 10]], np.int32))
            if out["done"][0] and out["reward"][0] == 0.0:
                hits.append(cell)
            one.close()
        assert hits == SEED7_MINES


def below(draw, n):
    """uniform_int_distribution{0, n - 1} on 32-bit words: Lemire's method."""
    m = draw() * n
    if m & 0xFFFFFFFF < n:
        t = (2**32 - n) % n
        while m & 0xFFFFFFFF < t:
            m = draw() * n
    return m >> 32


def register_shuffle_model(draw):
    """The kernel's register-only shuffle (envpool_b200/csrc/jumanji.cu random_mines): only the
    first 10 positions are stored; from step 10 on, position i still holds i before its swap."""
    f = list(range(10))
    j = below(draw, 2)
    f[1], f[j] = f[j], f[1]
    for i in range(2, 100, 2):
        j, k = divmod(below(draw, (i + 1) * (i + 2)), i + 2)
        if i < 10:
            f[i], f[j] = f[j], f[i]
            f[i + 1], f[k] = f[k], f[i + 1]
        else:
            if j < 10:
                f[j] = i
            if k < 10:
                f[k] = i + 1
    return f


# (engine outputs from the read position, read position); a 0 word is rejected by Lemire's method
# for every range the shuffle draws from except 2 and the powers of two
SHUFFLE_CASES = {
    "seeded, fresh table": ([], 624),
    "rejection in the first pair draw": ([None, 0], 100),
    "two rejections mid-shuffle": ([None] * 25 + [0, 0], 100),
    "rejection in the last draw": ([None] * 49 + [0], 100),
    "table regenerated mid-shuffle": ([None, 0] + [None] * 20, 600),
    "no rejection for range 2": ([0], 100),
}


@pytest.mark.parametrize("case", sorted(SHUFFLE_CASES))
def test_shuffle_models_equal_libstdcxx(case):
    """The oracle's full shuffle and the register-only model against std::shuffle on crafted
    engine states: the same first 10 cells in the same order, and the engines at the same
    word afterwards."""
    from oracle.ms_lib import MinesweeperOracle, StdShuffle

    outputs, idx = SHUFFLE_CASES[case]
    mt, _ = crafted_state(outputs, idx=min(idx, 600), seed=5)
    std = StdShuffle()
    std.set(mt, idx)
    want = list(std.shuffle())
    after = std.next()
    orc = MinesweeperOracle(1, seed=0)
    orc.set_rng(0, mt, idx)
    assert list(orc.shuffle(0)) == want
    assert orc.draw(0) == after
    model = MinesweeperOracle(1, seed=0)
    model.set_rng(0, mt, idx)
    assert register_shuffle_model(lambda: model.draw(0)) == want[:10]
    assert model.draw(0) == after


def test_register_shuffle_model_over_many_seeds():
    from oracle.ms_lib import MinesweeperOracle

    n = 300
    full = MinesweeperOracle(n, seed=1000)
    model = MinesweeperOracle(n, seed=1000)
    for e in range(n):
        want = list(full.shuffle(e)[:10])
        assert register_shuffle_model(lambda: model.draw(e)) == want, e
        assert model.draw(e) == full.draw(e), e


# ------------------------------------------------------------------ Reveal by hand ------
def board_of(out):
    return out["obs:board"][0]


def click(orc, r, c):
    return orc.step(np.array([[r, c]], np.int32))


def mines_at(cells):
    m = np.zeros(100, np.int32)
    m[list(cells)] = 1
    return m


def test_reveal_corner_flood_stops_at_a_wall_of_numbers():
    """Mines fill column 3: clicking a corner floods columns 0..1 (count 0) and shows column 2's
    counts (2 at the top and bottom rows, 3 elsewhere); the rest stays unexplored."""
    from oracle.ms_lib import MinesweeperOracle

    orc = MinesweeperOracle(1, seed=0, mines=mines_at(range(3, 100, 10)))
    out = orc.reset()
    assert (board_of(out) == -1).all() and out["obs:num_mines"][0] == 10
    out = click(orc, 0, 0)
    want = np.full((10, 10), -1, np.int32)
    want[:, :2] = 0
    want[:, 2] = 3
    want[[0, 9], 2] = 2
    np.testing.assert_array_equal(board_of(out), want)
    np.testing.assert_array_equal(out["obs:action_mask"][0], want == -1)
    assert out["reward"][0] == 1.0 and not out["done"][0] and out["obs:step_count"][0] == 1
    out = click(orc, 5, 2)                           # an explored cell: invalid, episode ends
    np.testing.assert_array_equal(board_of(out), want)
    assert out["reward"][0] == 0.0 and out["done"][0]


def test_reveal_full_flood_solves_the_board():
    """One mine in the middle: a corner click reveals all 99 other cells and solves the board."""
    from oracle.ms_lib import MinesweeperOracle

    orc = MinesweeperOracle(1, seed=0, mines=mines_at([55]))
    orc.reset()
    out = click(orc, 9, 0)
    b = board_of(out)
    assert b[5, 5] == -1 and (b[4:7, 4:7][np.arange(9).reshape(3, 3) != 4] == 1).all()
    assert (b >= 0).sum() == 99 and b[b >= 0].sum() == 8
    assert out["reward"][0] == 1.0 and out["done"][0] and out["obs:num_mines"][0] == 1


def test_reveal_mine_click_shows_its_count():
    from oracle.ms_lib import MinesweeperOracle

    orc = MinesweeperOracle(1, seed=0, mines=mines_at([0, 1, 10]))
    orc.reset()
    out = click(orc, 0, 0)                            # a mine with 2 mined neighbours
    b = board_of(out)
    assert b[0, 0] == 2 and (b.ravel()[1:] == -1).all()
    assert out["reward"][0] == 0.0 and out["done"][0]
    out = orc.step(np.array([[-7, INT32_MAX]], np.int32))   # the reset row: action ignored
    assert out["step_type"][0] == 0
    out = click(orc, 1, 1)                            # a number: only that cell
    b = board_of(out)
    assert b[1, 1] == 3 and (b >= 0).sum() == 1 and not out["done"][0]


def test_reveal_on_a_set_board_expands_only_through_unexplored_zeros():
    """A board with explored cells inside the zero region: the flood does not pass through
    them (Reveal visits unexplored cells only)."""
    from oracle.ms_lib import MinesweeperOracle

    orc = MinesweeperOracle(1, seed=0, mines=mines_at([99]))
    orc.reset()
    board = np.full((10, 10), -1, np.int32)
    board[:, 4] = 0                                   # an explored wall splitting the board
    orc.set_board(0, board)
    out = click(orc, 0, 0)
    b = board_of(out)
    assert (b[:, :4] == 0).all() and (b[:, 4] == 0).all() and (b[:, 5:] == -1).all()
    assert not out["done"][0]


# ---------------------------------------------------------------- spec and registry ------
def test_spec_keys_defaults_alias_and_spaces(engine_built):
    import envpool_b200 as ep
    from envpool_b200.jumanji import jumanji_envpool as jm

    S = jm._MinesweeperEnvSpec
    assert S._config_keys[10:] == ["minesweeper_mine_locations", "minesweeper_replay_boards",
                                   "minesweeper_replay_rewards", "minesweeper_replay_done"]
    assert S._default_config_values[10:] == ("", "", "", "")
    assert list(S._state_keys) == ["info:env_id", "info:players.env_id", "elapsed_step", "done",
                                   "reward", "discount", "step_type", "trunc", "obs:board",
                                   "obs:action_mask", "obs:num_mines", "obs:step_count"]
    assert list(S._action_keys) == ["env_id", "players.env_id", "action"]
    ids = ep.list_all_envs()
    assert "Minesweeper-v0" in ids and "Jumanji/Minesweeper-v0" in ids
    for tid in ("Minesweeper-v0", "Jumanji/Minesweeper-v0"):
        spec = ep.make_spec(tid, num_envs=3)
        assert spec.config.max_episode_steps == 90
        assert spec.config.minesweeper_mine_locations == ""
        st = dict(zip(spec._state_keys, spec._state_spec))
        assert st["obs:board"][1] == [10, 10] and st["obs:board"][2] == (-1, 8)
        assert np.dtype(st["obs:board"][0]) == np.int32
        assert st["obs:action_mask"][1] == [10, 10]
        assert np.dtype(st["obs:action_mask"][0]) == np.bool_
        assert st["obs:num_mines"][1] == [] and st["obs:num_mines"][2] == (0, 99)
        assert st["obs:step_count"][1] == [] and st["obs:step_count"][2] == (0, 90)
        act = dict(zip(spec._action_keys, spec._action_spec))["action"]
        assert np.dtype(act[0]) == np.int32 and act[1] == [-1, 2] and act[2] == (0, 9)


def test_spaces_follow_the_reference_data_transforms(engine_built):
    """What envpool/python/data.py makes of these specs: the shape [-1, 2] action is no
    discrete range (it has 2 elements), so a Box(0, 9, (2,), int32) and a dm BoundedArray; the
    scalar int observations are Discrete; the bool mask is MultiBinary."""
    import envpool_b200 as ep

    spec = ep.make_spec("Minesweeper-v0", num_envs=2)
    space = spec.observation_space
    assert isinstance(space, dict) and hasattr(space, "spaces")
    assert list(space.keys()) == ["board", "action_mask", "num_mines", "step_count"]
    assert space["board"].shape == (10, 10) and space["board"].dtype == np.int32
    assert type(space["action_mask"]).__name__ == "MultiBinary"
    assert space["action_mask"].shape == (10, 10)
    assert space["num_mines"].n == 100 and space["step_count"].n == 91
    act = spec.action_space
    assert type(act).__name__ == "Box" and act.shape == (2,) and act.dtype == np.int32
    assert (np.asarray(act.low) == 0).all() and (np.asarray(act.high) == 9).all()
    dm = spec.action_spec()
    assert tuple(dm.shape) == (2,) and dm.dtype == np.int32
    assert int(np.asarray(dm.minimum).max()) == 0 and int(np.asarray(dm.maximum).min()) == 9
    assert list(spec.observation_spec()._fields) == ["env_id", "players", "board",
                                                     "action_mask", "num_mines", "step_count"]


@pytest.mark.parametrize("kw", [
    dict(minesweeper_mine_locations="1,x"),
    dict(minesweeper_mine_locations=",5"),
    dict(minesweeper_mine_locations="99999999999"),
    dict(minesweeper_replay_boards="0,9"),
    dict(minesweeper_replay_boards="-2"),
    dict(minesweeper_replay_boards="1,,2"),
    dict(minesweeper_replay_boards="0", minesweeper_replay_rewards="0.5,x"),
    dict(minesweeper_replay_rewards="1e40"),
])
def test_malformed_strings_and_out_of_range_cells_raise_value_error(engine_built, kw):
    import envpool_b200 as ep

    with pytest.raises(ValueError):
        ep.make_spec("Minesweeper-v0", num_envs=2, **kw)


def test_strings_the_reference_accepts_are_accepted(engine_built):
    import envpool_b200 as ep

    ep.make_spec("Minesweeper-v0", num_envs=2, minesweeper_mine_locations="5, 7,3x,-1,100,",
                 minesweeper_replay_boards=",".join(["8"] * 3200 + ["x"]),
                 minesweeper_replay_rewards="1.5e0, -inf,nan", minesweeper_replay_done="yes,,1")
