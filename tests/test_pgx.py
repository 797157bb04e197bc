"""CPU: the PGX TicTacToe-v1 / ConnectFour-v1 checkers and boundary.  The C restatement
(oracle/pgx_oracle.c) against the fixtures recorded from the reference (tests/golden/pgx/) and,
where build() made it, against the reference's own thread pool (oracle/_ref) with odd
players.env_id mappings; the seed-7 known answer and pgx_deterministic_test.py's sequences; a
search that reaches every class of (state, action); the pybind classes' keys, specs and
defaults; and how EnvPoolMixin fills in players.env_id."""
import glob
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pgx_lib  # noqa: E402
from oracle.pgx_lib import ACTIONS, BOARD, PgxOracle, PgxRef, first_player_actions  # noqa: E402

GAMES = ["TicTacToe", "ConnectFour"]
FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "pgx", "*.npz")))
needs_ref = pytest.mark.skipif(not pgx_lib.ref_available(),
                               reason="oracle/_ref/libpgx_ref.so not built (no envpool checkout)")


def assert_same(got, want, ctx):
    for k, w in want.items():
        assert got[k].shape == w.shape and got[k].dtype == w.dtype, (ctx, k)
        assert np.array_equal(got[k], w), f"{ctx}: `{k}` differs"


def test_fixtures_cover_every_game_and_case():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert names == {f"{g}_{c}" for g in GAMES for c in ("random", "legal", "collide", "sequence")}


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_equals_fixture(path):
    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    data = {k: z[k] for k in z.files if k not in ("meta", "action")}
    orc = PgxOracle(meta["game"], meta["num_envs"], seed=meta["seed"])
    assert_same(orc.reset(), {k: v[0] for k, v in data.items()}, "reset")
    for t, a in enumerate(z["action"]):
        assert_same(orc.step(a), {k: v[t + 1] for k, v in data.items()}, f"step {t}")
    # the quirk the fixtures pin: player 1's discount is 0 on every row
    assert not data["discount"][:, 1::2].any()


@needs_ref
@pytest.mark.parametrize("game", GAMES)
def test_oracle_equals_ref_with_odd_player_rows(game):
    """Permuted env rows, permuted and duplicated player rows: each env acts with its first
    player row, and rows come back in submission order."""
    n = 96
    rng = np.random.default_rng(3)
    ref, orc = PgxRef(game, n, seed=12), PgxOracle(game, n, seed=12)
    assert_same(ref.reset(), orc.reset(), "reset")
    for t in range(400):
        ids = rng.permutation(n).astype(np.int32)
        pids = np.concatenate([ids, ids[rng.integers(0, n, size=int(rng.integers(0, n)))]])
        pids = pids[rng.permutation(len(pids))].astype(np.int32)
        acts = rng.integers(-1, ACTIONS[game] + 1, size=len(pids)).astype(np.int32)
        acts[rng.random(len(pids)) < 0.02] = np.iinfo(np.int32).min
        assert_same(ref.step(acts, ids, pids),
                    orc.step(first_player_actions(ids, pids, acts), ids), f"step {t}")


def mt19937_first(seed):
    """The first output of std::mt19937(seed) (init_genrand, one twist of word 0, tempering)."""
    mt = [seed & 0xffffffff]
    for i in range(1, 398):
        mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & 0xffffffff)
    y = (mt[0] & 0x80000000) | (mt[1] & 0x7fffffff)
    v = mt[397] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
    v ^= v >> 11
    v ^= (v << 7) & 0x9d2c5680
    v ^= (v << 15) & 0xefc60000
    v ^= v >> 18
    return v


@pytest.mark.parametrize("game", GAMES)
def test_seed_7_current_player(game):
    out = PgxOracle(game, 16, seed=7).reset()
    want = np.array([mt19937_first(7 + e) & 1 for e in range(16)], np.int32)
    assert mt19937_first(5489) == 3499211612  # std::mt19937's documented first output
    assert np.array_equal(out["info:current_player"], want)
    assert out["info:current_player"][0] == 1 and set(want.tolist()) == {0, 1}


@pytest.mark.parametrize("game,seq", [("TicTacToe", [0, 3, 1, 4, 2]),
                                      ("ConnectFour", [0, 1, 0, 1, 0, 1, 0])])
def test_deterministic_sequence(game, seq):
    """pgx_deterministic_test.py's sequences: the first mover completes a line on the last move."""
    n = 4
    orc = PgxOracle(game, n, seed=7)
    out = orc.reset()
    first = out["info:current_player"].copy()
    for t, a in enumerate(seq):
        out = orc.step(np.full(n, a, np.int32))
        assert out["done"].all() == (t == len(seq) - 1)
    r = out["reward"].reshape(n, 2)
    assert np.array_equal(r[np.arange(n), first], np.ones(n, np.float32))
    assert np.array_equal(r[np.arange(n), 1 - first], -np.ones(n, np.float32))
    assert not out["discount"].reshape(n, 2).any() and (out["step_type"] == 2).all()
    assert out["info:legal_action_mask"].all()  # a finished game's mask is all true
    board = out["info:board"]
    if game == "TicTacToe":
        assert (board[:, 0] == 0).all()  # colour 0 moves first: row 0 is its line
    else:
        assert (board[:, 2:, 0] == 0).all()  # four of colour 0 at the bottom of column 0


TTT_LINES = [(0, 1, 2), (3, 4, 5), (6, 7, 8), (0, 3, 6), (1, 4, 7), (2, 5, 8), (0, 4, 8), (2, 4, 6)]


def c4_win_directions(board, color):
    dirs = set()
    for r in range(6):
        for c in range(7):
            for d, (dr, dc) in enumerate(((1, 0), (0, 1), (1, 1), (1, -1))):
                if all(0 <= r + dr * k < 6 and 0 <= c + dc * k < 7 and
                       board[r + dr * k, c + dc * k] == color for k in range(4)):
                    dirs.add(d)
    return dirs


@pytest.mark.parametrize("game", GAMES)
def test_every_state_action_class_is_reached(game):
    """Random play with mostly legal moves reaches a win on every TicTacToe line and in every
    ConnectFour direction, draws, moves on occupied cells / into full columns and out-of-range
    actions; the same stream through the reference (when built) gives the same rows."""
    n, A = 512, ACTIONS[game]
    rng = np.random.default_rng(8)
    orc = PgxOracle(game, n, seed=1)
    ref = PgxRef(game, n, seed=1) if pgx_lib.ref_available() else None
    prev = orc.reset()
    if ref is not None:
        assert_same(ref.reset(), prev, "reset")
    seen = {}
    for t in range(600):
        mask = prev["info:legal_action_mask"]
        legal = np.argmax(np.where(mask, rng.random(mask.shape), -1), axis=1)
        wild = rng.integers(-2, A + 2, size=n)
        a = np.where(rng.random(n) < 0.93, legal, wild).astype(np.int32)
        out = orc.step(a)
        if ref is not None:
            assert_same(ref.step(a), out, f"step {t}")
        stepped = prev["done"] == 0
        for e in np.flatnonzero(stepped):
            if a[e] < 0 or a[e] >= A:
                seen["out of range"] = True
            elif not mask[e, a[e]]:
                seen["occupied cell" if game == "TicTacToe" else "full column"] = True
            elif out["done"][e]:
                r = out["reward"][2 * e:2 * e + 2]
                if not r.any():
                    seen["draw"] = True
                else:
                    mover = prev["info:current_player"][e]
                    assert r[mover] == 1 and r[1 - mover] == -1
                    b = out["info:board"][e]
                    color = b.ravel()[a[e]] if game == "TicTacToe" else \
                        b[:, a[e]][b[:, a[e]] >= 0][0]
                    if game == "TicTacToe":
                        for i, line in enumerate(TTT_LINES):
                            if all(b.ravel()[j] == color for j in line):
                                seen[f"line {i}"] = True
                    else:
                        for d in c4_win_directions(b, color):
                            seen[f"direction {d}"] = True
        prev = out
    want = {"out of range", "draw"} | (
        {"occupied cell"} | {f"line {i}" for i in range(8)} if game == "TicTacToe"
        else {"full column"} | {f"direction {d}" for d in range(4)})
    assert want <= set(seen), sorted(want - set(seen))


@pytest.mark.parametrize("game", GAMES)
def test_pybind_keys_specs_and_defaults(game):
    from envpool_b200.pgx import pgx_envpool as ext

    S = getattr(ext, f"_{game}EnvSpec")
    P = getattr(ext, f"_{game}EnvPool")
    r, c = BOARD[game]
    keys = ["info:env_id", "info:players.env_id", "elapsed_step", "done", "reward", "discount",
            "step_type", "trunc", "obs", "info:board", "info:current_player",
            "info:legal_action_mask", "info:players.id"]
    assert list(S._state_keys) == keys and list(P._state_keys) == keys
    assert list(S._action_keys) == ["env_id", "players.env_id", "action"]
    assert list(S._config_keys)[-1] == "task"
    task = "tic_tac_toe" if game == "TicTacToe" else "connect_four"
    assert S._default_config_values[-1] == task
    spec = S(S._default_config_values)
    st = dict(zip(keys, spec._state_spec))
    assert st["obs"][0] == np.bool_ and st["obs"][1] == [-1, r, c, 2]
    assert st["info:board"][1] == [r, c] and st["info:current_player"][1] == []
    assert st["info:legal_action_mask"][1] == [ACTIONS[game]]
    assert st["info:players.id"][1] == [-1] and st["info:players.id"][2] == (0, 1)
    for k in ("info:players.env_id", "reward", "discount"):
        assert st[k][1] == [-1]
    act = spec._action_spec[2]
    assert act[1] == [-1] and act[2] == (0, ACTIONS[game] - 1)


@pytest.mark.parametrize("game", GAMES)
def test_registration(game):
    import envpool_b200

    task = f"{game}-v1"
    assert task in envpool_b200.list_all_envs()
    spec = envpool_b200.make_spec(task)
    assert spec.config.max_num_players == 2
    assert spec.config.max_episode_steps == np.iinfo(np.int32).max
    assert spec.config.task == ("tic_tac_toe" if game == "TicTacToe" else "connect_four")


def _mixin(n, players=2):
    import envpool_b200
    from envpool_b200.python.envpool import EnvPoolMixin

    spec = envpool_b200.make_spec("TicTacToe-v1", num_envs=n, max_num_players=players)

    class Pool(EnvPoolMixin):
        pass

    p = Pool.__new__(Pool)
    p._spec = spec._spec if hasattr(spec, "_spec") else spec
    p.spec = spec
    return p


def test_players_env_id_resolution():
    p = _mixin(4)
    ids = np.arange(4, dtype=np.int32)
    a = np.zeros(4, np.int32)
    # one action per env: players.env_id = env_id
    assert np.array_equal(p._from(a)[1], ids)
    # two per env and nothing cached: each env id repeated
    assert np.array_equal(p._from(np.zeros(8, np.int32))[1], np.repeat(ids, 2))
    # an explicit players.env_id wins
    explicit = np.array([3, 3, 0, 1, 2], np.int32)
    got = p._from({"action": np.zeros(5, np.int32), "players.env_id": explicit})
    assert np.array_equal(got[1], explicit)
    # the last recv's player rows of the envs, in env_id order
    p._last_players_env_id = np.array([2, 2, 0, 0, 1, 1, 3, 3], np.int32)
    got = p._from(np.zeros(4, np.int32), env_id=np.array([1, 3], np.int32))
    assert np.array_equal(got[1], [1, 1, 3, 3])
    # neither: the row count must be a multiple of the env count, at most max_num_players each
    with pytest.raises(RuntimeError, match="Cannot infer"):
        p._from(np.zeros(5, np.int32), env_id=np.array([0, 1], np.int32))
    with pytest.raises(RuntimeError, match="exceeds max_num_players"):
        p._from(np.zeros(6, np.int32), env_id=np.array([1, 2], np.int32))
    p._check_action(p._from(np.zeros(8, np.int32)))  # player-row actions pass the check


def test_single_player_pools_keep_players_env_id_equal_to_env_id():
    import envpool_b200
    from envpool_b200.python.envpool import EnvPoolMixin

    spec = envpool_b200.make_spec("CartPole-v1", num_envs=3)

    class Pool(EnvPoolMixin):
        pass

    p = Pool.__new__(Pool)
    p._spec, p.spec = spec._spec if hasattr(spec, "_spec") else spec, spec
    got = p._from(np.zeros(2, np.int32), env_id=np.array([2, 0], np.int32))
    assert np.array_equal(got[0], [2, 0]) and np.array_equal(got[1], [2, 0])


def test_sharded_pool_takes_the_two_player_kinds():
    """ShardedPool forwards TicTacToe / ConnectFour (per-player columns ride in the shard's slab
    like any other) and holds max_num_players to 2; the check runs before any device work."""
    from envpool_b200.sharded import ShardedPool

    for task in ("TicTacToe-v1", "ConnectFour-v1"):
        with pytest.raises(ValueError, match="max_num_players must be 2"):
            ShardedPool(task, 8, max_num_players=1)


def test_pool_layout_fixture_covers_every_two_player_case():
    from envpool_b200 import _capi

    sys.path[:0] = [GOLDEN, os.path.join(GOLDEN, "pgx")]
    from make_pgx_pool_layouts import FIXTURE, cases

    assert list(_capi.TWO_PLAYER_KINDS) == GAMES
    with open(FIXTURE) as f:
        want = json.load(f)
    assert sorted(want) == sorted(dict(cases(_capi.TWO_PLAYER_KINDS)))
    # per-player columns lead with the player dimension; their rows cover both players
    ttt = want["TicTacToe/f64/iopt=0/n=1000"]
    keys = {k["name"]: (k["shape"], k["row_bytes"]) for k in ttt["keys"]}
    assert keys["obs"] == ([2, 3, 3, 2], 36) and keys["reward"] == ([2], 8)
    assert keys["info:board"] == ([3, 3], 36) and ttt["bytes_per_env_step"] == 151
    assert want["ConnectFour/f64/iopt=0/n=1000"]["bytes_per_env_step"] == 445
