"""CPU: the PGX Chess and GardnerChess checkers and boundary.  The C restatement
(oracle/chess_oracle.c) against the reference's own thread pool (oracle/_ref/libchess_ref.so, where
build() made it) over legal-random play to the step limit and over random labels with permuted
players.env_id rows; the off-board label rule; perft from the initial position, independent of
the reference; the pybind classes' keys and specs, the registration, the ValueError on
max_num_players and the engine's kind table."""
import glob
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from pgx_chess_scripts import CLASSES, hand_written, reached, scripts
from test_pgx import assert_same, mt19937_first

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import chess_lib  # noqa: E402
from oracle.chess_lib import GAMES, MAX_STEPS, actions, first_player_actions  # noqa: E402
from oracle.chess_lib import ChessOracle as Oracle, ChessRef as Ref  # noqa: E402

TASK_ID = {g: f"{g}-v1" for g in GAMES}
I32 = np.iinfo(np.int32)
# perft from the initial position: leaf counts at depth 1..5
PERFT = [20, 400, 8902, 197281, 4865609]
FIXTURE_DIR = os.path.join(GOLDEN, "pgx", "chess")
FIXTURES = sorted(glob.glob(os.path.join(FIXTURE_DIR, "*.npz")))
needs_ref = pytest.mark.skipif(not chess_lib.ref_available(),
                               reason="oracle/_ref/libchess_ref.so not built (no envpool checkout)")


def load_fixture(path):
    """(meta, {key: [T + 1, rows, ...]} with the mask unpacked and obs rebuilt from its bit-packed
    planes and per-row scalar channels, actions [T, n]); obs only at data["obs_steps"]."""
    sys.path.insert(0, FIXTURE_DIR)
    from make_chess_golden import unpack_obs

    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    data = {k: z[k] for k in z.files if k not in ("meta", "obs_planes", "obs_scalars")}
    data["obs"] = unpack_obs(z["obs_planes"], z["obs_scalars"], meta["obs_shape"][2])
    assert list(data["obs"].shape) == meta["obs_shape"]
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


def test_fixtures_cover_every_game_and_case():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert names == {f"{g}_{c}" for g in GAMES for c in ("random", "legal", "collide", "sequence")}
    assert sum(os.path.getsize(p) for p in FIXTURES) < 4 << 20


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_equals_fixture(path):
    meta, data = load_fixture(path)
    orc = Oracle(meta["game"], meta["num_envs"], seed=meta["seed"])
    assert_same(orc.reset(), row(data, 0), "reset")
    for t, a in enumerate(data["action"]):
        assert_same(orc.step(a), row(data, t + 1), f"step {t}")


@pytest.mark.parametrize("game", list(GAMES))
def test_scripts_reach_every_class(game):
    """Every class, and each script its own class (the checkmates: either player losing)."""
    found = reached(game)
    assert set(CLASSES[game]) <= set(found), sorted(set(CLASSES[game]) - set(found))
    for name in scripts(game):
        if name.startswith("checkmate"):
            assert {"checkmate_player0_loses", "checkmate_player1_loses"} <= \
                {k for k, v in found.items() if name in v}, name
        else:
            assert name in found[name], name


def test_sequence_fixture_holds_every_on_board_script():
    """The reference recorded every script but those with an off-board label."""
    for game in GAMES:
        meta, _ = load_fixture(os.path.join(FIXTURE_DIR, f"{game}_sequence.npz"))
        off = [k for k in hand_written(game) if k.startswith("off_board")]
        assert meta["num_envs"] == len(scripts(game)) - len(off), game


def legal_fast(rng, mask):
    return np.argmax(np.where(mask, rng.random(mask.shape), -1.0), axis=1).astype(np.int32)


def out_of_range(game):
    return np.array([-1, -2, actions(game), actions(game) + 1, I32.min, I32.max], np.int32)


def noisy(game, rng, mask, on_board, share=0.03):
    """A legal label, else (share) any label whose target lies on the board, else (share / 8) an
    out-of-range one.  The reference's own Step writes board[-1] for labels whose target lies off
    the board, so those are never sent to it (test_off_board_labels checks the oracle's rule)."""
    n = mask.shape[0]
    a = legal_fast(rng, mask)
    u = rng.random(n)
    a = np.where(u < share, on_board[rng.integers(0, len(on_board), n)], a)
    return np.where(u < share / 8, out_of_range(game)[rng.integers(0, 6, n)], a).astype(np.int32)


@needs_ref
@pytest.mark.parametrize("game", list(GAMES))
def test_oracle_equals_ref_legal_play_to_the_step_limit(game):
    """256 envs of legal-random play until at least one game of each seed ends on the step limit;
    obs, masks, keys and counters over whole games."""
    n = 256
    orc, ref = Oracle(game, n, seed=9), Ref(game, n, seed=9)
    want = orc.reset()
    assert_same(ref.reset(), want, "reset")
    rng = np.random.default_rng(1)
    limit = 0
    for t in range(MAX_STEPS[game] + 2):
        a = legal_fast(rng, want["info:legal_action_mask"])
        want = orc.step(a)
        assert_same(ref.step(a), want, f"step {t}")
        limit += int((want["done"] & (want["elapsed_step"] == MAX_STEPS[game])).sum())
    assert limit > 0


@needs_ref
@pytest.mark.parametrize("game", list(GAMES))
def test_oracle_equals_ref_random_labels_with_permuted_player_rows(game):
    n = 32
    rng = np.random.default_rng(3)
    orc, ref = Oracle(game, n, seed=12), Ref(game, n, seed=12)
    on_board = np.flatnonzero(orc.on_board())
    prev = orc.reset()
    assert_same(ref.reset(), prev, "reset")
    mask = prev["info:legal_action_mask"].copy()
    for t in range(300):
        ids = rng.permutation(n).astype(np.int32)
        pids = ids[rng.permutation(n)]
        acts = noisy(game, rng, mask[pids], on_board, 0.1)
        want = orc.step(first_player_actions(ids, pids, acts), ids)
        assert_same(ref.step(acts, ids, pids), want, f"step {t}")
        mask[ids] = want["info:legal_action_mask"]


def _label(game, frm, plane):
    return frm * chess_lib.PLANES[game] + plane


@pytest.mark.parametrize("game", list(GAMES))
def test_off_board_labels(game):
    """A label whose target lies off the board: the piece leaves its square, nothing lands, the
    target reads as empty.  A pawn on square 1 counts it as a double pawn move in Chess
    (en_passant 0 before the flip, 7 after it); a knight's leaves halfmove_count at 1."""
    S = chess_lib.SIZE[game]
    orc = Oracle(game, 4, seed=3)
    out = orc.reset()
    start = out["info:board"].copy()
    # a pawn on square 1 (column 0, row 1) with underpromotion planes 0 and 4; the knight on
    # square S jumping (-1, -2) (plane 9 + 8 (S - 1)); the rook on square 0 moving one column to
    # the left (plane 9 + 2 (S - 1) + S - 2)
    knight_off = 9 + 8 * (S - 1)
    rook_off = 9 + 2 * (S - 1) + (S - 2)
    acts = np.array([_label(game, 1, 0), _label(game, S, knight_off), _label(game, 0, rook_off),
                     _label(game, 1, 4)], np.int32)
    on = orc.on_board()
    assert not on[acts].any()
    out = orc.step(acts)
    assert out["done"].all() and (out["elapsed_step"] == 1).all()
    r = out["reward"].reshape(4, 2)
    assert (r.sum(1) == 0).all() and (np.abs(r) == 1).all()
    assert out["info:legal_action_mask"].all()
    assert (out["info:halfmove_count"] == [0, 1, 1, 0]).all()
    # the mover's piece is gone; the board is flipped: square p of the mover is -board[flip(p)]
    flipped = -start[:, ::-1, :]
    for e, sq in enumerate([1, S, 0, 1]):
        b = flipped[e].copy()
        row, col = S - 1 - sq % S, sq // S
        b[S - 1 - row, col] = 0  # the flip maps row r to S - 1 - r
        assert np.array_equal(out["info:board"][e], b), e
    if game == "Chess":
        assert (out["info:en_passant"] == [7, -1, -1, 7]).all()
        assert out["info:castling_rights"][2].tolist() == [[True, True], [False, True]]


def test_perft_from_the_initial_position():
    """Every ply-d position reached by stepping the oracle through all legal sequences: the legal
    masks' popcounts over the envs not done sum to perft(d + 1), d = 0..4 (published counts)."""
    seqs = np.zeros((1, 0), np.int32)
    for d in range(5):
        total, children = 0, []
        for c0 in range(0, len(seqs), 16384):
            chunk = seqs[c0:c0 + 16384]
            orc = Oracle("Chess", len(chunk), seed=1, obs=False)
            out = orc.reset()
            for k in range(d):
                out = orc.step(chunk[:, k])
            live = ~out["done"]
            mask = out["info:legal_action_mask"] & live[:, None]
            total += int(mask.sum())
            if d < 4:
                e, a = np.nonzero(mask)
                children.append(np.concatenate([chunk[e], a[:, None].astype(np.int32)], 1))
            orc.close()
        assert total == PERFT[d], (d, total)
        if d < 4:
            seqs = np.concatenate(children)


@pytest.mark.parametrize("game", list(GAMES))
def test_reset_player_order_and_initial_position(game):
    S = chess_lib.SIZE[game]
    out = Oracle(game, 16, seed=7).reset()
    want = np.array([mt19937_first(7 + e) & 1 for e in range(16)], np.int32)
    assert np.array_equal(out["info:current_player"], want)
    assert (out["info:turn"] == 0).all() and (out["info:fullmove_count"] == 1).all()
    assert out["info:legal_action_mask"].sum(1).tolist() == [20 if game == "Chess" else 7] * 16
    obs = out["obs"].reshape(16, 2, S, S, -1)
    assert (obs[..., 12::14][..., :8] == 1).all() and (obs[..., 13::14][..., :8] == 0).all()
    assert not obs[..., 14:112].reshape(16, 2, S, S, 7, 14)[..., :12].any()  # empty history
    mover = obs[np.arange(16), want]
    other = obs[np.arange(16), 1 - want]
    assert (mover[..., 112] == 0).all() and (other[..., 112] == 1).all()


def test_pybind_keys_specs_and_defaults():
    from envpool_b200.pgx import pgx_envpool as ext

    for game in GAMES:
        S, P = getattr(ext, f"_{game}EnvSpec"), getattr(ext, f"_{game}EnvPool")
        keys = [k for k, *_ in chess_lib.keys(game)]
        assert list(S._state_keys) == keys and list(P._state_keys) == keys
        assert list(S._action_keys) == ["env_id", "players.env_id", "action"]
        assert list(S._config_keys)[-1] == "task"
        task = "chess" if game == "Chess" else "gardner_chess"
        assert tuple(S._default_config_values)[-1] == task
        spec = S(tuple(S._default_config_values))
        st = dict(zip(keys, spec._state_spec))
        size, A = chess_lib.SIZE[game], actions(game)
        assert st["obs"][0] == np.float32
        assert st["obs"][1] == [-1, size, size, chess_lib.CHANNELS[game]]
        assert st["info:board"][1] == [size, size]
        assert st["info:current_player"][2] == (0, 1) and st["info:turn"][2] == (0, 1)
        assert st["info:legal_action_mask"][1] == [A]
        assert st["info:players.id"][1] == [-1] and st["info:players.id"][2] == (0, 1)
        if game == "Chess":
            assert st["info:castling_rights"][1] == [2, 2]
            assert st["info:en_passant"][2] == (-1, 63)
        act = spec._action_spec[2]
        assert act[1] == [-1] and act[2] == (0, A - 1)


@pytest.mark.parametrize("game", list(GAMES))
def test_registration(game):
    import envpool_b200

    task = TASK_ID[game]
    assert task in envpool_b200.list_all_envs()
    c = envpool_b200.make_spec(task).config
    assert c.max_num_players == 2
    assert c.task == ("chess" if game == "Chess" else "gardner_chess")


@pytest.mark.parametrize("game", list(GAMES))
@pytest.mark.parametrize("players", [1, 3])
def test_max_num_players_must_be_two(game, players):
    import envpool_b200

    with pytest.raises(ValueError, match="max_num_players must be 2"):
        envpool_b200.make_gymnasium(TASK_ID[game], num_envs=2, max_num_players=players)


def test_sharded_pool_holds_max_num_players_to_two():
    from envpool_b200.sharded import ShardedPool

    for task in TASK_ID.values():
        for players in (1, 3):
            with pytest.raises(ValueError, match="max_num_players must be 2"):
                ShardedPool(task, 8, max_num_players=players)


def test_capi_tables():
    from envpool_b200 import _capi

    assert _capi.CHESS_KINDS == {"Chess": 21, "GardnerChess": 22}
    assert not set(_capi.CHESS_KINDS) & set(_capi.ALL_KINDS)
    assert not set(_capi.CHESS_KINDS) & set(_capi.GO_KINDS)
    assert not set(_capi.CHESS_KINDS.values()) & set(_capi.ALL_KINDS.values())
    assert not set(_capi.CHESS_KINDS.values()) & set(_capi.GO_KINDS.values())
