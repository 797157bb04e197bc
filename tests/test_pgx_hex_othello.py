"""CPU: the PGX Hex-v1 / Othello-v1 checkers and boundary.  The C restatement
(oracle/hex_othello_oracle.c) against the fixtures recorded from the reference
(tests/golden/pgx/hex_othello/) and, where build() made it, against the reference's own thread
pool (oracle/_ref) with odd players.env_id mappings; the seed-7 known answer; the seeded search
that reaches every class of (state, action); the pybind classes' keys, specs and defaults, the
registration and ShardedPool's player check."""
import glob
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from pgx_hex_othello_scripts import CLASSES, scripts
from test_pgx import assert_same, mt19937_first

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import hex_othello_lib  # noqa: E402
from oracle.hex_othello_lib import ACTIONS, BOARD, PLANES, first_player_actions  # noqa: E402
from oracle.hex_othello_lib import HexOthelloOracle as Oracle, HexOthelloRef as Ref  # noqa: E402

GAMES = ["Hex", "Othello"]
CASES = ("random", "legal", "collide", "sequence")
FIXTURE_DIR = os.path.join(GOLDEN, "pgx", "hex_othello")
FIXTURES = sorted(glob.glob(os.path.join(FIXTURE_DIR, "*.npz")))
TASK = {"Hex": "hex", "Othello": "othello"}
needs_ref = pytest.mark.skipif(not hex_othello_lib.ref_available(),
                               reason="oracle/_ref/libhex_othello_ref.so not built (no envpool checkout)")


def test_fixtures_cover_every_game_and_case():
    assert list(hex_othello_lib.GAMES) == GAMES
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert names == {f"{g}_{c}" for g in GAMES for c in CASES}


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_equals_fixture(path):
    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    data = {k: z[k] for k in z.files if k not in ("meta", "action")}
    orc = Oracle(meta["game"], meta["num_envs"], seed=meta["seed"])
    assert_same(orc.reset(), {k: v[0] for k, v in data.items()}, "reset")
    for t, a in enumerate(z["action"]):
        assert_same(orc.step(a), {k: v[t + 1] for k, v in data.items()}, f"step {t}")
    assert not data["discount"][:, 1::2].any()
    assert not data["trunc"].any()  # no max_episode_steps: INT_MAX


@needs_ref
@pytest.mark.parametrize("game", GAMES)
def test_oracle_equals_ref_with_odd_player_rows(game):
    n = 96
    rng = np.random.default_rng(3)
    ref, orc = Ref(game, n, seed=12), Oracle(game, n, seed=12)
    prev = orc.reset()
    assert_same(ref.reset(), prev, "reset")
    mask = prev["info:legal_action_mask"].copy()  # each env's mask, by env id
    for t in range(400):
        ids = rng.permutation(n).astype(np.int32)
        pids = np.concatenate([ids, ids[rng.integers(0, n, size=int(rng.integers(0, n)))]])
        pids = pids[rng.permutation(len(pids))].astype(np.int32)
        acts = rng.integers(-1, ACTIONS[game] + 1, size=len(pids))
        legal = np.argmax(np.where(mask, rng.random(mask.shape), -1), axis=1)[pids]
        acts = np.where(rng.random(len(pids)) < 0.9, legal, acts).astype(np.int32)
        acts[rng.random(len(pids)) < 0.01] = np.iinfo(np.int32).min
        want = orc.step(first_player_actions(ids, pids, acts), ids)
        assert_same(ref.step(acts, ids, pids), want, f"step {t}")
        mask[ids] = want["info:legal_action_mask"]


@pytest.mark.parametrize("game", GAMES)
def test_seed_7_current_player(game):
    out = Oracle(game, 16, seed=7).reset()
    want = np.array([mt19937_first(7 + e) & 1 for e in range(16)], np.int32)
    assert np.array_equal(out["info:current_player"], want)
    if game == "Othello":
        mask = out["info:legal_action_mask"]
        assert (np.flatnonzero(mask[0]) == [19, 26, 37, 44]).all()
    else:  # the first word picks player_order_: colour 0 moves first, plane 2 reads 0 for it
        obs = out["obs"].reshape(16, 2, 11, 11, 4)
        assert not obs[np.arange(16), want, :, :, 2].any()
        assert obs[np.arange(16), 1 - want, :, :, 2].all()


@pytest.mark.parametrize("game", GAMES)
def test_search_reaches_every_class(game):
    """The seeded search of pgx_hex_othello_scripts reaches every class; each script replays
    to its class in a fresh oracle, the same through the reference when it is built."""
    found = scripts(game)
    assert set(CLASSES[game]) <= set(found), sorted(set(CLASSES[game]) - set(found))
    n = len(found)
    orc = Oracle(game, n, seed=4)
    ref = Ref(game, n, seed=4) if hex_othello_lib.ref_available() else None
    out = orc.reset()
    if ref is not None:
        assert_same(ref.reset(), out, "reset")
    acts = list(found.values())
    for t in range(max(len(s) for s in acts)):
        mask = out["info:legal_action_mask"]
        a = np.array([s[t] if t < len(s) else int(np.argmax(mask[i]))
                      for i, s in enumerate(acts)], np.int32)
        out = orc.step(a)
        if ref is not None:
            assert_same(ref.step(a), out, f"step {t}")
        for i, s in enumerate(acts):
            if t == len(s) - 1:
                assert not out["step_type"][i] == 0, list(found)[i]


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
    assert S._default_config_values[-1] == TASK[game]
    spec = S(S._default_config_values)
    st = dict(zip(keys, spec._state_spec))
    assert st["obs"][0] == np.bool_ and st["obs"][1] == [-1, r, c, PLANES[game]]
    assert st["info:board"][1] == [r, c] and st["info:current_player"][1] == []
    assert st["info:legal_action_mask"][1] == [ACTIONS[game]]
    assert st["info:players.id"][1] == [-1] and st["info:players.id"][2] == (0, 1)
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
    assert spec.config.task == TASK[game]


def test_sharded_pool_holds_max_num_players_to_two():
    from envpool_b200.sharded import ShardedPool

    for task in ("Hex-v1", "Othello-v1"):
        for players in (1, 3):
            with pytest.raises(ValueError, match="max_num_players must be 2"):
                ShardedPool(task, 8, max_num_players=players)
    with pytest.raises(ValueError, match="max_num_players"):
        ShardedPool("CartPole-v1", 8, max_num_players=2)


def test_capi_resolves_every_table():
    from envpool_b200 import _capi

    assert _capi.TWO_PLAYER_KINDS_2 == {"Hex": 16, "Othello": 17}
    assert _capi.ALL_KINDS == {**_capi.KINDS, **_capi.TWO_PLAYER_KINDS, **_capi.TWO_PLAYER_KINDS_2}


def test_pool_layout_fixture_covers_every_case():
    from envpool_b200 import _capi

    sys.path[:0] = [GOLDEN, os.path.join(GOLDEN, "pgx")]
    from make_pgx_pool_layouts import cases

    with open(os.path.join(FIXTURE_DIR, "pool_layouts.json")) as f:
        want = json.load(f)
    assert sorted(want) == sorted(dict(cases(_capi.TWO_PLAYER_KINDS_2)))
    hexk = {k["name"]: (k["shape"], k["row_bytes"]) for k in want["Hex/f64/iopt=0/n=1000"]["keys"]}
    assert hexk["obs"] == ([2, 11, 11, 4], 968) and hexk["info:legal_action_mask"] == ([122], 122)
    oth = {k["name"]: (k["shape"], k["row_bytes"]) for k in want["Othello/f64/iopt=0/n=1000"]["keys"]}
    assert oth["obs"] == ([2, 8, 8, 2], 256) and oth["info:board"] == ([8, 8], 256)
