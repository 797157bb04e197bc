"""CPU: the PGX Go checkers and boundary.  The C restatement (oracle/go_oracle.c) against the
fixtures recorded from the reference (tests/golden/pgx/go/) and, where build() made it, against
the reference's own thread pool (oracle/_ref) with permuted players.env_id rows and every
configuration; the scripts of pgx_go_scripts.py reach every class at every board size; the seed-7
answer; the pybind class's keys, specs and defaults, the ValueError cases, the registration and
ShardedPool's player check."""
import glob
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from pgx_go_scripts import CLASSES, reached, scripts
from test_pgx import assert_same, mt19937_first

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import go_lib  # noqa: E402
from oracle.go_lib import GAMES, actions, first_player_actions  # noqa: E402
from oracle.go_lib import GoOracle as Oracle, GoRef as Ref  # noqa: E402

FIXTURE_DIR = os.path.join(GOLDEN, "pgx", "go")
FIXTURES = sorted(glob.glob(os.path.join(FIXTURE_DIR, "*.npz")))
TASK_ID = {g: f"{g}-v1" for g in GAMES}
needs_ref = pytest.mark.skipif(not go_lib.ref_available(),
                               reason="oracle/_ref/libgo_ref.so not built (no envpool checkout)")


def load_fixture(path):
    """(meta, {key: [T + 1, rows, ...]} with obs and the mask unpacked, actions [T, n]); obs
    only at meta's `obs_steps` (data["obs_steps"])."""
    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    data = {k: z[k] for k in z.files if k not in ("meta",)}
    shape = meta["obs_shape"]
    data["obs"] = np.unpackbits(data["obs"], axis=-1, count=int(np.prod(shape[2:]))) \
        .astype(bool).reshape(shape)
    shape = meta["mask_shape"]
    data["info:legal_action_mask"] = np.unpackbits(
        data["info:legal_action_mask"], axis=-1, count=shape[2]).astype(bool).reshape(shape)
    return meta, data


def row(data, t):
    """The expected columns of record t (obs only where the fixture keeps it)."""
    out = {k: v[t] for k, v in data.items() if k not in ("action", "obs", "obs_steps")}
    hit = np.flatnonzero(data["obs_steps"] == t)
    if hit.size:
        out["obs"] = data["obs"][hit[0]]
    return out


def pool_kwargs(meta):
    return {k: meta[k] for k in ("komi", "max_terminal_steps") if k in meta}


def test_fixtures_cover_every_game_and_case():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    want = set()
    for g, s in GAMES.items():
        want |= {f"{g}_{c}" for c in ("random", "legal", "collide", "sequence", "komi_0",
                                      "komi_-3.5", "komi_0.5", "mts_1", "mts_5",
                                      f"mts_{2 * s * s}")}
    assert names == want


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_equals_fixture(path):
    meta, data = load_fixture(path)
    orc = Oracle(meta["game"], meta["num_envs"], seed=meta["seed"], **pool_kwargs(meta))
    assert_same(orc.reset(), row(data, 0), "reset")
    for t, a in enumerate(data["action"]):
        assert_same(orc.step(a), row(data, t + 1), f"step {t}")
    assert not data["discount"][:, 1::2].any()
    assert not data["trunc"].any()


def test_legal_fixtures_run_games_to_max_terminal_steps():
    """The `legal` and `mts_2S^2` records hold games that end on the step limit, with every
    hash of the history stored."""
    for g, s in GAMES.items():
        for case in ("legal", f"mts_{2 * s * s}"):
            _, data = load_fixture(os.path.join(FIXTURE_DIR, f"{g}_{case}.npz"))
            assert (data["done"] & (data["elapsed_step"] == 2 * s * s)).any(), (g, case)


@pytest.mark.parametrize("game", list(GAMES))
@pytest.mark.parametrize("komi", ["0", "-3.5", "0.5"])
def test_komi_fixtures_hold_scored_double_pass_ends(game, komi):
    """Each komi record holds double-pass ends that the area comparison scores, won by each
    colour; komi 0 holds one at equal areas, which white wins (black - komi > white is strict).
    So the fixture tests pin the kernel's komi handling to the reference."""
    _, data = load_fixture(os.path.join(FIXTURE_DIR, f"{game}_komi_{komi}.npz"))
    assert (data["obs_steps"] == np.arange(len(data["done"]))).all()  # obs at every record
    n = data["done"].shape[1]
    ends = np.argwhere(data["done"] & (data["info:consecutive_pass_count"] == 2))
    winners, equal_white = set(), False
    for t, e in ends:
        obs = data["obs"][t].reshape(n, 2, -1, 17)
        black = 0 if not obs[e, 0, 0, 16] else 1  # plane 16: the player's colour is white
        r = data["reward"][t].reshape(n, 2)[e]
        assert r[black] == -r[1 - black] != 0
        ba, wa = data["info:black_area"][t, e], data["info:white_area"][t, e]
        assert (r[black] > 0) == (ba - float(komi) > wa), (t, e)
        winners.add("black" if r[black] > 0 else "white")
        equal_white |= ba == wa and r[black] < 0
    assert winners == {"black", "white"}, winners
    assert equal_white or komi != "0"


@needs_ref
@pytest.mark.parametrize("game", list(GAMES))
@pytest.mark.parametrize("komi,mts", [(7.5, 0), (0.0, 0), (-3.5, 5), (0.5, 1), (7.5, -1)])
def test_oracle_equals_ref_with_permuted_player_rows(game, komi, mts):
    """GoEnv::Step CHECKs one action per env, so every env has exactly one player row."""
    n = 24
    mts = 2 * GAMES[game] ** 2 if mts < 0 else mts
    rng = np.random.default_rng(3)
    ref = Ref(game, n, seed=12, komi=komi, max_terminal_steps=mts)
    orc = Oracle(game, n, seed=12, komi=komi, max_terminal_steps=mts)
    prev = orc.reset()
    assert_same(ref.reset(), prev, "reset")
    mask = prev["info:legal_action_mask"].copy()
    A = actions(game)
    for t in range(150):
        ids = rng.permutation(n).astype(np.int32)
        pids = ids[rng.permutation(n)]
        acts = rng.integers(-1, A + 1, size=len(pids))
        legal = np.argmax(np.where(mask, rng.random(mask.shape), -1), axis=1)[pids]
        acts = np.where(rng.random(len(pids)) < 0.97, legal, acts).astype(np.int32)
        acts[rng.random(len(pids)) < 0.003] = np.iinfo(np.int32).min
        want = orc.step(first_player_actions(ids, pids, acts), ids)
        assert_same(ref.step(acts, ids, pids), want, f"step {t}")
        mask[ids] = want["info:legal_action_mask"]


@pytest.mark.parametrize("game", list(GAMES))
def test_scripts_reach_every_class(game):
    found = reached(game)
    assert set(CLASSES) <= set(found), sorted(set(CLASSES) - set(found))


@needs_ref
@pytest.mark.parametrize("game", list(GAMES))
def test_scripts_on_the_reference(game):
    sc = list(scripts(game).values())
    n = len(sc)
    orc, ref = Oracle(game, n, seed=4), Ref(game, n, seed=4)
    out = orc.reset()
    assert_same(ref.reset(), out, "reset")
    for t in range(max(len(s) for s in sc) + 2):
        mask = out["info:legal_action_mask"]
        a = np.array([s[t] if t < len(s) else int(np.argmax(mask[i])) for i, s in enumerate(sc)],
                     np.int32)
        out = orc.step(a)
        assert_same(ref.step(a), out, f"step {t}")


@pytest.mark.parametrize("game", list(GAMES))
def test_config_classes(game):
    """max_terminal_steps ends a game on its step, both player orders occur, and komi 0 at equal
    areas gives the game to white (black - komi > white is strict)."""
    S = GAMES[game]
    A = S * S
    orc = Oracle(game, 4, seed=5, max_terminal_steps=5)
    orc.reset()
    for t in range(5):
        out = orc.step(np.full(4, t, np.int32))
    assert out["done"].all() and (out["elapsed_step"] == 5).all()
    assert not out["info:is_psk"].any() and (out["info:consecutive_pass_count"] == 0).all()
    assert (out["reward"] != 0).all()
    first = Oracle(game, 16, seed=7).reset()["info:current_player"]
    assert set(first.tolist()) == {0, 1}
    orc = Oracle(game, 16, seed=7, komi=0.0)
    orc.reset()
    orc.step(np.full(16, A, np.int32))
    out = orc.step(np.full(16, A, np.int32))
    assert out["done"].all() and (out["info:black_area"] == A).all()
    assert (out["info:white_area"] == A).all()
    black = np.where(first == 0, 0, 1)  # player order: the player to move first plays black
    r = out["reward"].reshape(16, 2)
    assert (r[np.arange(16), black] == -1).all() and (r[np.arange(16), 1 - black] == 1).all()


@pytest.mark.parametrize("game", list(GAMES))
def test_seed_7_player_order(game):
    out = Oracle(game, 16, seed=7).reset()
    want = np.array([(mt19937_first(7 + e) >> 1) & 1 for e in range(16)], np.int32)
    assert np.array_equal(out["info:current_player"], want)
    S = GAMES[game]
    assert out["info:legal_action_mask"].all()
    assert not out["obs"][..., :16].any()
    obs = out["obs"].reshape(16, 2, S, S, 17)
    assert not obs[np.arange(16), want, :, :, 16].any()  # the first mover plays black (colour 0)
    assert obs[np.arange(16), 1 - want, :, :, 16].all()
    assert (out["info:black_area"] == S * S).all() and (out["info:white_area"] == S * S).all()
    assert (out["info:ko"] == -1).all()


def test_pybind_keys_specs_and_defaults():
    from envpool_b200.pgx import pgx_envpool as ext

    S, P = ext._GoEnvSpec, ext._GoEnvPool
    keys = ["info:env_id", "info:players.env_id", "elapsed_step", "done", "reward", "discount",
            "step_type", "trunc", "obs", "info:board", "info:current_player",
            "info:legal_action_mask", "info:ko", "info:is_psk", "info:consecutive_pass_count",
            "info:black_area", "info:white_area", "info:players.id"]
    assert list(S._state_keys) == keys and list(P._state_keys) == keys
    assert list(S._action_keys) == ["env_id", "players.env_id", "action"]
    assert list(S._config_keys)[-6:] == ["board_size", "komi", "history_length",
                                         "max_terminal_steps", "rules", "task"]
    assert tuple(S._default_config_values)[-6:] == (19, 7.5, 8, 0, "pgx", "go_19x19")
    for size in GAMES.values():
        conf = list(S._default_config_values)
        conf[-6] = size
        spec = S(tuple(conf))
        st = dict(zip(keys, spec._state_spec))
        A = size * size
        assert st["obs"][0] == np.bool_ and st["obs"][1] == [-1, size, size, 17]
        assert st["info:board"][1] == [size, size] and st["info:board"][2] == (-1, 1)
        assert st["info:current_player"][2] == (0, 1)
        assert st["info:legal_action_mask"][1] == [A + 1]
        assert st["info:ko"][2] == (-1, A - 1)
        assert st["info:is_psk"][0] == np.bool_
        assert st["info:players.id"][1] == [-1] and st["info:players.id"][2] == (0, 1)
        act = spec._action_spec[2]
        assert act[1] == [-1] and act[2] == (0, A)


@pytest.mark.parametrize("kwargs,match", [
    (dict(board_size=7), "board_size 7"), (dict(board_size=21), "board_size 21"),
    (dict(history_length=4), "history_length"), (dict(max_terminal_steps=-1), "max_terminal"),
    (dict(max_terminal_steps=163), "max_terminal"), (dict(rules="chinese"), "chinese"),
    (dict(rules="japanese"), "japanese")])
def test_unaccelerated_options_raise(kwargs, match):
    import envpool_b200

    with pytest.raises(ValueError, match=match):
        envpool_b200.make_spec("Go9x9-v1", **kwargs)


def test_accepted_options():
    import envpool_b200

    for task, size in (("Go9x9-v1", 9), ("Go13x13-v1", 13), ("Go19x19-v1", 19)):
        for mts in (0, 1, 2 * size * size):
            spec = envpool_b200.make_spec(task, max_terminal_steps=mts, rules="tromp_taylor",
                                          komi=-3.5)
            assert spec.config.max_terminal_steps == mts and spec.config.komi == -3.5


@pytest.mark.parametrize("game", list(GAMES))
def test_registration(game):
    import envpool_b200

    task = TASK_ID[game]
    assert task in envpool_b200.list_all_envs()
    spec = envpool_b200.make_spec(task)
    c = spec.config
    assert c.max_num_players == 2 and c.board_size == GAMES[game]
    assert (c.komi, c.history_length, c.max_terminal_steps, c.rules) == (7.5, 8, 0, "pgx")
    assert c.task == f"go_{GAMES[game]}x{GAMES[game]}"
    assert not any(t.startswith("ChineseGo") for t in envpool_b200.list_all_envs())


def test_sharded_pool_holds_max_num_players_to_two():
    from envpool_b200.sharded import ShardedPool

    for task in TASK_ID.values():
        for players in (1, 3):
            with pytest.raises(ValueError, match="max_num_players must be 2"):
                ShardedPool(task, 8, max_num_players=players)
        with pytest.raises(ValueError, match="cannot carry"):
            ShardedPool(task, 8, rules="chinese")


def test_capi_tables():
    from envpool_b200 import _capi

    assert _capi.GO_KINDS == {"Go9x9": 18, "Go13x13": 19, "Go19x19": 20}
    assert not set(_capi.GO_KINDS) & set(_capi.ALL_KINDS)
    assert "epb_go_config" in _capi.ABI_SYMBOLS
