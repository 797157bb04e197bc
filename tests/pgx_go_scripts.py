"""Action scripts for PGX Go that reach every class of (state, action) the kernel in csrc/go.cu
treats differently, at each board size: hand-written sequences, plus the positional-superko
endings a seeded search of legal play found (`search_psk`, pinned in
tests/golden/pgx/go/psk_scripts.json by make_go_golden.py).

`scripts(game)` returns {name: [action, ...]}: the actions of one episode from its reset.  Go's
board dynamics do not depend on the seed (the reset draw only picks which player plays black), so
a script replays in any env of any pool.  `classes(game, prev, out, e, a)` names the classes one
step of env e reached; tests/test_pgx_go.py asserts that the scripts reach every class in
CLASSES, and tests/test_gpu_pgx_go.py replays them on the device.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.go_lib import GAMES, GoOracle  # noqa: E402

I32 = np.iinfo(np.int32)
PSK_FILE = os.path.join(HERE, "golden", "pgx", "go", "psk_scripts.json")
CLASSES = ["single-stone capture", "multi-stone capture", "multi-chain capture", "ko set",
           "ko point played, capture applied", "suicide", "occupied own", "occupied opponent",
           "action -1", "action pass", "action S^2+1", "action INT_MIN", "action INT_MAX",
           "double pass, black wins", "double pass, white wins", "psk end",
           "empty region touching neither colour"]
# the classes that need a configured pool or several resets: tests/test_pgx_go.py
CONFIG_CLASSES = ["max_terminal_steps end", "both player orders", "strict komi at equal areas"]


def hand_written(game):
    S = GAMES[game]
    A = S * S

    def p(r, c):
        return r * S + c

    return {
        "single capture": [p(0, 1), p(0, 0), p(1, 0)],
        "two-stone capture": [p(1, 0), p(0, 0), p(1, 1), p(0, 1), p(0, 2)],
        "two chains at once": [p(1, 0), p(0, 0), p(1, 2), p(0, 2), p(0, 3), A, p(0, 1)],
        # black takes the white stone on (1, 1) from (1, 2); white retakes at once: the ko point
        "ko": [p(0, 1), p(0, 2), p(1, 0), p(1, 3), p(2, 1), p(2, 2), A, p(1, 1), p(1, 2), p(1, 1)],
        "suicide": [p(0, 1), p(5, 5), p(1, 0), p(0, 0)],
        "own stone": [p(0, 0), p(1, 1), p(0, 0)],
        "opponent stone": [p(0, 0), p(0, 0)],
        "minus one": [-1],
        "past the pass": [A + 1],
        "int min": [int(I32.min)],
        "int max": [int(I32.max)],
        "pass pass": [A, A],
        "black then pass pass": [p(S // 2, S // 2), A, A],
    }


def scripts(game):
    out = hand_written(game)
    with open(PSK_FILE) as f:
        out["psk"] = json.load(f)[game]
    return out


def _components(cells, S):
    """connected components (4-neighbour) of a boolean [S * S] array"""
    seen = np.zeros_like(cells)
    sizes = []
    for start in np.flatnonzero(cells):
        if seen[start]:
            continue
        stack, size = [start], 0
        seen[start] = True
        while stack:
            c = stack.pop()
            size += 1
            r, q = divmod(c, S)
            for rr, qq in ((r - 1, q), (r + 1, q), (r, q - 1), (r, q + 1)):
                n = rr * S + qq
                if 0 <= rr < S and 0 <= qq < S and cells[n] and not seen[n]:
                    seen[n] = True
                    stack.append(n)
        sizes.append(size)
    return sizes


def classes(game, prev, out, e, a):
    """The classes env e reached stepping from `prev` to `out` with action a (not a reset)."""
    S = GAMES[game]
    A = S * S
    got = []
    cur = int(prev["info:current_player"][e])
    my = -1 if prev["obs"][2 * e + cur][0, 0, 16] else 1  # the mover's stones
    before = prev["info:board"][e].ravel()
    after = out["info:board"][e].ravel()
    special = {-1: "action -1", A: "action pass", A + 1: "action S^2+1",
               int(I32.min): "action INT_MIN", int(I32.max): "action INT_MAX"}
    if a in special:
        got.append(special[a])
    elif 0 <= a < A:
        if before[a] == my:
            got.append("occupied own")
        elif before[a] == -my:
            got.append("occupied opponent")
        elif a != prev["info:ko"][e] and not prev["info:legal_action_mask"][e][a]:
            got.append("suicide")
        sizes = _components((before == -my) & (after == 0), S)
        if sizes:
            got.append("single-stone capture" if sizes == [1] else "multi-stone capture")
            if len(sizes) > 1:
                got.append("multi-chain capture")
            if a == prev["info:ko"][e]:
                got.append("ko point played, capture applied")
        if out["info:ko"][e] >= 0 and not out["done"][e]:
            got.append("ko set")
    if out["done"][e]:
        if a == A and out["info:consecutive_pass_count"][e] == 2:
            black_player = cur if my == 1 else 1 - cur
            won = out["reward"][2 * e + black_player] > 0
            got.append("double pass, black wins" if won else "double pass, white wins")
        if out["info:is_psk"][e]:
            got.append("psk end")
    if (not after.any() and a == A and out["info:black_area"][e] == A and
            out["info:white_area"][e] == A):
        got.append("empty region touching neither colour")
    return got


def reached(game, **pool_kwargs):
    """{class: script name} for the scripts replayed on the oracle, one env each."""
    sc = scripts(game)
    names = list(sc)
    n = len(names)
    orc = GoOracle(game, n, seed=3, **pool_kwargs)
    prev = orc.reset()
    found = {}
    for t in range(max(len(s) for s in sc.values())):
        mask = prev["info:legal_action_mask"]
        a = np.array([sc[k][t] if t < len(sc[k]) else int(np.argmax(mask[i]))
                      for i, k in enumerate(names)], np.int32)
        out = orc.step(a)
        for i, k in enumerate(names):
            if t < len(sc[k]) and not prev["done"][i]:
                for c in classes(game, prev, out, i, int(a[i])):
                    found.setdefault(c, k)
        prev = out
    return found


def search_psk(game, n, seed, steps=100_000):
    """Legal play without passes in n envs (seeded) until an episode ends in positional superko:
    the actions of that episode."""
    A = GAMES[game] ** 2
    rng = np.random.default_rng(seed)
    orc = GoOracle(game, n, seed=1)
    prev = orc.reset()
    hist = [[] for _ in range(n)]
    for _ in range(steps):
        m = prev["info:legal_action_mask"].copy()
        m[:, A] = ~m[:, :A].any(1)
        a = np.argmax(np.where(m, rng.random(m.shape), -1), axis=1).astype(np.int32)
        out = orc.step(a)
        for e in range(n):
            if prev["done"][e]:
                hist[e] = []
                continue
            hist[e].append(int(a[e]))
            if out["done"][e] and out["info:is_psk"][e]:
                return hist[e]
        prev = out
    raise RuntimeError(f"{game}: no superko in {steps} steps")
