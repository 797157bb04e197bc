"""PGX Chess / GardnerChess action scripts that reach every rule class the kernel must reproduce.

`scripts(game)` -> {class: [label, ...]}: one episode from the initial position per class, each
ending with the step that shows it.  The illegal, off-board and out-of-range scripts are written
by hand (one label from the initial position); the others come from `search(game)`, a seeded
search over legal-random play of the oracle, and are stored in tests/golden/pgx/chess/scripts.json
(tests/golden/pgx/chess/make_chess_golden.py writes it).  Only the first player depends on the
env's seed, so the scripts hold under any seed; `reached(game)` replays every script under seeds
giving both player orders and returns the classes each one shows (`classify`), which is how a
checkmate reaches both "player 0 loses" and "player 1 loses".
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import chess_lib  # noqa: E402
from oracle.chess_lib import ChessOracle  # noqa: E402

SCRIPTS_JSON = os.path.join(HERE, "golden", "pgx", "chess", "scripts.json")
I32 = np.iinfo(np.int32)
PER_PLAYER = ("reward", "discount", "info:players.env_id", "info:players.id", "obs")
DIRS = {0: "forward", 1: "capture_up", -1: "capture_down"}  # column change of a promotion

_PROMOTIONS = [f"promote_{p}_{d}" for p in "qrbn" for d in DIRS.values()]
_ENDINGS = ["checkmate_player0_loses", "checkmate_player1_loses", "stalemate", "fifty_moves",
            "threefold_repetition", "insufficient_kings", "insufficient_minor_piece",
            "insufficient_bishops_one_colour", "step_limit"]
_ILLEGAL = ["illegal_empty_square", "illegal_opponent_piece", "illegal_blocked_move",
            "off_board_underpromotion", "off_board_ray", "off_board_knight", "out_of_range_-1",
            "out_of_range_actions", "out_of_range_int_min", "out_of_range_int_max"]
CLASSES = {
    "Chess": ["castle_queen_side", "castle_king_side", "castle_queen_side_square_8_attacked",
              "castle_refused_16_attacked", "castle_refused_24_attacked",
              "castle_refused_32_attacked", "castle_refused_40_attacked",
              "castle_refused_48_attacked", "rights_lost_king_move", "rights_lost_rook_move",
              "rights_lost_rook_captured", "en_passant_from_ep_minus_9",
              "en_passant_from_ep_plus_7", "en_passant_refused_king_attacked",
              "en_passant_pinned_along_the_row",
              "illegal_castle_label"] + _PROMOTIONS + _ENDINGS + _ILLEGAL,
    "GardnerChess": _PROMOTIONS + _ENDINGS + _ILLEGAL,
}
SEARCH = {"Chess": (4096, 1, 1400), "GardnerChess": (2048, 2, 900)}  # envs, seed, steps


def _pos(info_board, S):
    """[n, S, S] info:board rows -> [n, S^2] boards indexed by square col * S + row."""
    p = np.arange(S * S)
    return info_board[:, S - 1 - p % S, p // S]


def hand_written(game):
    S, P, A = chess_lib.SIZE[game], chess_lib.PLANES[game], chess_lib.actions(game)
    R = S - 1
    out = {
        "illegal_empty_square": [2 * P + 9 + R],          # square 2 (empty) one row up
        "illegal_opponent_piece": [(S - 1) * P + 9 + R - 1],  # the other side's rook one down
        "illegal_blocked_move": [0 * P + 9 + R + 1],      # the rook through its own pawn
        "off_board_underpromotion": [1 * P + 0],          # pawn on square 1, not on row S - 2
        "off_board_ray": [0 * P + 9 + 2 * R + R - 1],     # the rook one column left of column 0
        "off_board_knight": [S * P + 9 + 8 * R],          # the knight on square S, (-1, -2)
        "out_of_range_-1": [-1], "out_of_range_actions": [A],
        "out_of_range_int_min": [int(I32.min)], "out_of_range_int_max": [int(I32.max)],
    }
    if game == "Chess":
        out["illegal_castle_label"] = [2364]  # the queen-side castle with pieces in between
    return out


def classify(game, orc, pre, acts, post, square_8_attacked):
    """The classes each env's step shows: pre / post the oracle's outputs before and after the
    step, square_8_attacked [n] bool of the pre position."""
    S, P, A = chess_lib.SIZE[game], chess_lib.PLANES[game], chess_lib.actions(game)
    n = len(acts)
    b0, b1 = _pos(pre["info:board"], S), _pos(post["info:board"], S)
    out = [set() for _ in range(n)]
    for e in range(n):
        a = int(acts[e])
        if pre["done"][e]:
            continue
        found = out[e]
        if a < 0 or a >= A:
            found.add({-1: "out_of_range_-1", A: "out_of_range_actions",
                       int(I32.min): "out_of_range_int_min",
                       int(I32.max): "out_of_range_int_max"}.get(a, "out_of_range"))
            continue
        f, plane = a // P, a % P
        to = orc.label_target(a)
        legal = bool(pre["info:legal_action_mask"][e, a])
        piece = int(b0[e, f])
        if not legal:
            if to < 0:
                found.add("off_board_underpromotion" if plane < 9 else
                          "off_board_knight" if plane >= 9 + 8 * (S - 1) else "off_board_ray")
            elif piece == 0:
                found.add("illegal_empty_square")
            elif piece < 0:
                found.add("illegal_opponent_piece")
            elif game == "Chess" and a in (2364, 2367) and piece == 6:
                found.add("illegal_castle_label")
            else:
                found.add("illegal_blocked_move")
            continue
        # legal moves
        if piece == 1 and f % S == S - 2:
            dc = (to // S) - (f // S)
            kind = "q" if plane >= 9 else "rbn"[plane // 3]
            found.add(f"promote_{kind}_{DIRS[dc]}")
        if game == "Chess":
            rights0 = pre["info:castling_rights"][e]
            if piece == 6 and f == 32 and to in (16, 48):
                found.add("castle_queen_side" if to == 16 else "castle_king_side")
                if to == 16 and square_8_attacked[e]:
                    found.add("castle_queen_side_square_8_attacked")
            if rights0[0].any() and ((piece == 6 and f == 32) or (piece == 4 and f in (0, 56))):
                lost = rights0[0] & ~post["info:castling_rights"][e][1]
                if lost.any():
                    found.add("rights_lost_king_move" if piece == 6 else "rights_lost_rook_move")
            if to in (7, 63) and b0[e, to] == -4 and rights0[1][0 if to == 7 else 1]:
                found.add("rights_lost_rook_captured")
            ep = int(pre["info:en_passant"][e])
            if piece == 1 and ep >= 0 and to == ep:
                found.add("en_passant_from_ep_minus_9" if f == ep - 9 else "en_passant_from_ep_plus_7")
        ended = orc.ended(e)
        if post["done"][e]:
            r = post["reward"].reshape(n, 2)[e]
            if ended & 1 and ended & 2:
                found.add(f"checkmate_player{int(np.argmin(r))}_loses")
            elif ended & 1:
                found.add("stalemate")
            if ended & 4:
                found.add("fifty_moves")
            if ended & 16:
                found.add("threefold_repetition")
            if ended & 32:
                found.add("step_limit")
            if ended & 8:
                pieces = int((b1[e] != 0).sum())
                found.add("insufficient_kings" if pieces == 2 else
                          "insufficient_minor_piece" if pieces == 3 else
                          "insufficient_bishops_one_colour")
    return out


def position_classes(game, orc, out, ids=None):
    """Classes of a position itself (castling or en passant refused), before its move; env i of
    the batch is oracle env ids[i]."""
    n = len(out["done"])
    res = [set() for _ in range(n)]
    if game != "Chess":
        return res
    P = 73
    b = _pos(out["info:board"], 8)
    for e in range(n):
        if out["done"][e]:
            continue
        env = e if ids is None else ids[e]
        x, rights, mask = b[e], out["info:castling_rights"][e][0], out["info:legal_action_mask"][e]
        if rights[0] and x[0] == 4 and x[8] == 0 and x[16] == 0 and x[24] == 0 and x[32] == 6:
            for sq in (16, 24, 32):
                if orc.attacked(env, sq):
                    res[e].add(f"castle_refused_{sq}_attacked")
        if rights[1] and x[32] == 6 and x[40] == 0 and x[48] == 0 and x[56] == 4:
            for sq in (32, 40, 48):
                if orc.attacked(env, sq):
                    res[e].add(f"castle_refused_{sq}_attacked")
        ep = int(out["info:en_passant"][e])
        if ep >= 1 and x[ep - 1] == -1:
            for f in (ep - 9, ep + 7):
                if 0 <= f < 64 and x[f] == 1:
                    label = next(f * P + pl for pl in range(9, P)
                                 if orc.label_target(f * P + pl) == ep)
                    if not mask[label]:
                        res[e].add("en_passant_refused_king_attacked")
                        king = np.flatnonzero(x == 6)
                        if len(king) and king[0] % 8 == (ep - 1) % 8:  # the pawns' row
                            res[e].add("en_passant_pinned_along_the_row")
    return res


def _square_8(game, orc, out, acts, ids):
    """Whether square 8 is attacked where a legal queen-side castle is about to be played."""
    res = np.zeros(len(acts), bool)
    if game == "Chess":
        for i, a in enumerate(acts):
            if a == 2364 and not out["done"][i] and out["info:legal_action_mask"][i, 2364]:
                res[i] = orc.attacked(ids[i], 8)
    return res


def run(game, episodes, env_seed):
    """Replay one script per env (then stop acting: the env keeps its last outputs); the classes
    each env's script showed, the position its last label leads to included."""
    n = len(episodes)
    orc = ChessOracle(game, n, seed=0, env_seed=np.asarray(env_seed, np.int32), obs=False)
    out = orc.reset()
    found = [set() for _ in range(n)]
    live = np.ones(n, bool)
    for t in range(max(len(s) for s in episodes) + 1):
        # the position after a script's last label is examined too (position classes)
        seen = np.flatnonzero(np.array([t <= len(s) for s in episodes]) & live)
        for i, c in enumerate(position_classes(
                game, orc, {k: v[seen] for k, v in out.items() if k not in PER_PLAYER}, seen)):
            found[seen[i]] |= c
        ids = np.flatnonzero(np.array([t < len(s) for s in episodes]) & live)
        if not len(ids):
            break
        pre = {k: v[ids] for k, v in out.items() if k not in PER_PLAYER}
        acts = np.array([episodes[e][t] for e in ids], np.int32)
        att8 = _square_8(game, orc, pre, acts, ids)
        post_ids = orc.step(acts, ids)
        cls = classify(game, _Sub(orc, ids), pre, acts, post_ids, att8)
        for i, e in enumerate(ids):
            found[e] |= cls[i]
            for k, v in post_ids.items():
                if k in ("reward", "discount", "info:players.env_id", "info:players.id"):
                    out[k].reshape(n, 2)[e] = v.reshape(len(ids), 2)[i]
                else:
                    out[k][e] = v[i]
        live[ids[post_ids["done"]]] = False
    return found


class _Sub:
    """The oracle seen through a batch of env ids (classify indexes envs by batch row)."""

    def __init__(self, orc, ids):
        self.orc, self.ids = orc, ids

    def ended(self, i):
        return self.orc.ended(self.ids[i])

    def label_target(self, a):
        return self.orc.label_target(a)

    def attacked(self, i, sq):
        return self.orc.attacked(self.ids[i], sq)


def search(game):
    """A seeded search over legal-random play; the first episode showing each class, up to and
    including that step."""
    n, seed, steps = SEARCH[game]
    want = set(CLASSES[game]) - set(hand_written(game))
    orc = ChessOracle(game, n, seed=seed, obs=False)
    rng = np.random.default_rng(seed)
    out = orc.reset()
    episode = [[] for _ in range(n)]
    found = {}
    for t in range(steps):
        if want <= set(found):
            break
        for e, c in enumerate(position_classes(game, orc, out)):
            for k in c - set(found):
                found[k] = list(episode[e])
        mask = out["info:legal_action_mask"]
        acts = np.argmax(np.where(mask, rng.random(mask.shape), -1.0), axis=1).astype(np.int32)
        att8 = _square_8(game, orc, out, acts, np.arange(n))
        post = orc.step(acts)
        cls = classify(game, orc, out, acts, post, att8)
        for e in range(n):
            if out["done"][e]:
                episode[e] = []
                continue
            episode[e].append(int(acts[e]))
            for k in cls[e] - set(found):
                found[k] = list(episode[e])
        out = post
    return {k: v for k, v in found.items() if k in want}


def scripts(game):
    with open(SCRIPTS_JSON) as f:
        found = json.load(f)[game]
    return {**found, **hand_written(game)}


def seeds_with_both_orders():
    """Two env seeds whose first player differs (bit 0 of the first mt19937 word)."""
    first = {}
    for s in range(64):
        first.setdefault(_mt_first(s) & 1, s)
    return [first[0], first[1]]


def _mt_first(seed):
    mt = [0] * 624
    mt[0] = seed & 0xffffffff
    for i in range(1, 624):
        mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xffffffff
    y = (mt[0] & 0x80000000) | (mt[1] & 0x7fffffff)
    v = mt[397] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
    v ^= v >> 11
    v ^= (v << 7) & 0x9d2c5680
    v ^= (v << 15) & 0xefc60000
    v ^= v >> 18
    return v


def reached(game):
    """{class: [script names showing it]} over every script replayed under both player orders."""
    sc = scripts(game)
    names = list(sc)
    s0, s1 = seeds_with_both_orders()
    found = run(game, [sc[k] for k in names] * 2, [s0] * len(names) + [s1] * len(names))
    out = {}
    for i, c in enumerate(found):
        for k in c:
            out.setdefault(k, set()).add(names[i % len(names)])
    return out
