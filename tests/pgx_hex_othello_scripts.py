"""A seeded search on the C restatement (oracle/hex_othello_oracle.c) for Hex and Othello action scripts
that reach every class of (state, action) the kernels in csrc/pgx.cu treat differently.

`scripts(game)` returns {class: [action, ...]}: the actions of one episode from its reset up to
and including the step that reached the class.  The board dynamics of both games do not depend
on the seed (the reset draw only picks which player moves first), so a script replays in any
env of any pool.  tests/test_pgx_hex_othello.py asserts that every class in CLASSES is reached;
tests/test_gpu_pgx_hex_othello.py replays the scripts on the device.
"""
import functools
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.hex_othello_lib import ACTIONS, HexOthelloOracle  # noqa: E402

I32 = np.iinfo(np.int32)
# the eight directions of board_games.h kOthelloShifts as (row, column) steps
DIRS = [(0, 1), (0, -1), (1, 0), (-1, 0), (1, -1), (-1, 1), (1, 1), (-1, -1)]
CLASSES = {
    "Hex": ["win colour 0", "win colour 1", "legal swap then win", "swap at step 0",
            "swap at step >= 2", "swap of a diagonal stone", "overwrite own stone",
            "overwrite opponent stone", "action -1", "action 122", "action INT_MIN",
            "action INT_MAX"],
    "Othello": [f"flip direction {d}" for d in range(8)] + [
        "no wrap from column 0", "no wrap from column 7", "forced pass", "double pass ends",
        "full board", "wipe-out", "mover wins", "mover loses", "draw", "illegal pass",
        "occupied cell that flips"],
}


def _hex_classes(prev, out, e, a, swapped):
    """Classes of Hex env e stepping from `prev` with action a (not a reset step)."""
    got = []
    mask = prev["info:legal_action_mask"][e]
    board = prev["info:board"][e].ravel()  # +1 the mover's stones, -1 the opponent's
    cur = prev["info:current_player"][e]
    color = int(prev["obs"][2 * e + cur][0, 0, 2])
    special = {-1: "action -1", 122: "action 122", int(I32.min): "action INT_MIN",
               int(I32.max): "action INT_MAX"}
    if a in special:
        got.append(special[a])
    elif a == 121:
        # the swap is legal at step 1 only; a running game has an empty board at step 0 only
        if not mask[121]:
            got.append("swap at step >= 2" if board.any() else "swap at step 0")
        occ = np.flatnonzero(board)
        if occ.size and occ[0] // 11 == occ[0] % 11:
            got.append("swap of a diagonal stone")
    elif board[a] == 1:
        got.append("overwrite own stone")
    elif board[a] == -1:
        got.append("overwrite opponent stone")
    elif out["done"][e] and out["reward"][2 * e:2 * e + 2].any():
        got.append(f"win colour {color}")
        if swapped:
            got.append("legal swap then win")
    return got


def _oth_line(board, r, c, dr, dc):
    """Cells captured from (r, c) along (dr, dc) by the +1 side of `board` (8x8)."""
    run = []
    rr, cc = r + dr, c + dc
    while 0 <= rr < 8 and 0 <= cc < 8 and board[rr, cc] == -1:
        run.append((rr, cc))
        rr, cc = rr + dr, cc + dc
    return run if (0 <= rr < 8 and 0 <= cc < 8 and board[rr, cc] == 1 and run) else []


def _oth_classes(prev, out, e, a, passed):
    got = []
    mask = prev["info:legal_action_mask"][e]
    board = prev["info:board"][e]  # +1 the mover's stones
    done = bool(out["done"][e])
    if a == 64:
        if not mask[64]:
            got.append("illegal pass")
        elif passed and done:
            got.append("double pass ends")
        elif not done:
            got.append("forced pass")
    elif 0 <= a < 64:
        r, c = divmod(a, 8)
        flips = [d for d, (dr, dc) in enumerate(DIRS) if _oth_line(board, r, c, dr, dc)]
        if board[r, c] != 0 and flips:
            got.append("occupied cell that flips")
        if mask[a]:
            got += [f"flip direction {d}" for d in flips]
            # a line that would capture if the row wrapped into the next (or previous) one
            flat = board.ravel()
            for step, col in ((1, 7), (-1, 0)):
                if c != col:
                    continue
                k, run = a + step, 0
                while 0 <= k < 64 and flat[k] == -1:
                    k, run = k + step, run + 1
                if run and 0 <= k < 64 and flat[k] == 1:
                    got.append(f"no wrap from column {col}")
    if done and mask[a if 0 <= a <= 64 else 0] and 0 <= a <= 64:
        nb = out["info:board"][e]  # the next mover's view: -1 the stones of the player who moved
        if (nb != 0).all():
            got.append("full board")
        if not (nb == 1).any():
            got.append("wipe-out")
        r = out["reward"][2 * e:2 * e + 2]
        mover = prev["info:current_player"][e]
        got.append("draw" if not r.any() else ("mover wins" if r[mover] > 0 else "mover loses"))
    return got


@functools.lru_cache(maxsize=None)
def _search(game, n=512, steps=1500, seed=0):
    rng = np.random.default_rng(seed)
    A = ACTIONS[game]
    orc = HexOthelloOracle(game, n, seed=seed + 1)
    prev = orc.reset()
    hist = [[] for _ in range(n)]
    flag = np.zeros(n, bool)  # Hex: a legal swap this episode; Othello: the last move passed
    found = {}
    specials = np.array([-1, A, I32.min, I32.max], np.int64)
    for t in range(steps):
        mask = prev["info:legal_action_mask"]
        legal = np.argmax(np.where(mask, rng.random(mask.shape), -1), axis=1)
        u = rng.random(n)
        a = legal.copy()
        a = np.where(u < 0.004, specials[rng.integers(0, 4, size=n)], a)
        if game == "Hex":
            a = np.where((u > 0.5) & mask[:, 121], 121, a)  # take the legal swap half the time
            a = np.where((u >= 0.004) & (u < 0.01), 121, a)
            occ = prev["info:board"].reshape(n, -1) != 0
            pick = np.argmax(np.where(occ, rng.random(occ.shape), -1), axis=1)
            a = np.where((u >= 0.01) & (u < 0.016) & occ.any(1), pick, a)
            a = np.where((u >= 0.016) & (u < 0.02) & ~occ.any(1), 0, a)
        else:
            a = np.where((u >= 0.004) & (u < 0.008), 64, a)
            occ = prev["info:board"].reshape(n, -1) != 0
            pick = np.argmax(np.where(occ, rng.random(occ.shape), -1), axis=1)
            a = np.where((u >= 0.008) & (u < 0.014), pick, a)
        a = a.astype(np.int32)
        out = orc.step(a)
        for e in range(n):
            if prev["done"][e]:
                hist[e] = []
                flag[e] = False
                continue
            hist[e].append(int(a[e]))
            if game == "Hex":
                cls = _hex_classes(prev, out, e, int(a[e]), flag[e])
                if a[e] == 121 and prev["info:legal_action_mask"][e, 121]:
                    flag[e] = True
            else:
                cls = _oth_classes(prev, out, e, int(a[e]), flag[e])
                flag[e] = a[e] == 64
            for c in cls:
                found.setdefault(c, list(hist[e]))
        prev = out
        if set(CLASSES[game]) <= set(found):
            break
    return found


def scripts(game):
    """{class: actions from a reset}, for every class the search reached."""
    return {c: list(s) for c, s in _search(game).items()}
