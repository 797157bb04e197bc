"""Record the PGX Hex-v1 / Othello-v1 fixtures from the reference's own thread pool.

    python tests/golden/pgx/hex_othello/make_hex_othello_golden.py   # needs oracle/_ref (build())

The same record as ../make_pgx_golden.py keeps for TicTacToe and ConnectFour, in the same .npz
format (`meta`, `action` [T, n], every state key as [T + 1, rows, ...]) and with its `random` and
`legal` policies, for every game of hex_othello_lib.GAMES.  Cases:
  random      actions over the whole int32 range (make_pgx_golden.policy)
  legal       a uniformly random legal action of each env (make_pgx_golden.policy)
  collide     Hex: the swap at step 0, at step 1 (legal) and later, a first stone on the diagonal
              (cell 0 or 60), moves onto occupied cells of either colour; Othello: moves onto
              occupied cells, passes while a move exists; legal moves otherwise
  sequence    pgx_deterministic_test.py's policy -- the legal actions' (3 step + 1) % count-th --
              for 30 steps, then the illegal cases of pgx_align_test.py (Hex 0, 0; Othello 0)
              and the policy again
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(HERE))))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle import hex_othello_lib  # noqa: E402
from make_pgx_golden import policy as pgx_policy  # noqa: E402

ILLEGAL = {"Hex": [0, 0], "Othello": [0]}
CASES = {"random": (32, 3, 200), "legal": (16, 5, 400), "collide": (32, 11, 200),
         "sequence": (8, 7, 40)}


def deterministic(mask, t):
    out = np.empty(len(mask), np.int32)
    for e, m in enumerate(mask):
        acts = np.flatnonzero(m)
        out[e] = acts[(t * 3 + 1) % acts.size]
    return out


def collide(game, rng, mask, out):
    n, A = mask.shape
    legal = np.argmax(np.where(mask, rng.random(mask.shape), -1), axis=1).astype(np.int32)
    occupied = out["info:board"].reshape(n, -1) != 0
    a = legal.copy()
    u = rng.random(n)
    for e in range(n):
        occ = np.flatnonzero(occupied[e])
        if occ.size and u[e] < 0.12:
            a[e] = rng.choice(occ)
        elif game == "Hex" and u[e] < 0.2:
            a[e] = 121
        elif game == "Hex" and not occ.size and u[e] < 0.5:
            a[e] = rng.choice([0, 60, 12, 5])  # a first stone on the diagonal, or off it
        elif game == "Hex" and mask[e, 121] and u[e] < 0.8:
            a[e] = 121
        elif game == "Othello" and u[e] < 0.2:
            a[e] = 64
    return a


def record(game, case):
    n, seed, T = CASES[case]
    rng = np.random.default_rng(seed)
    ref = hex_othello_lib.HexOthelloRef(game, n, seed=seed)
    outs = [ref.reset()]
    acts = []
    for t in range(T):
        mask = outs[-1]["info:legal_action_mask"]
        if case in ("random", "legal"):
            a = pgx_policy(case, game, rng, t, mask)
        elif case == "collide":
            a = collide(game, rng, mask, outs[-1])
        elif 30 <= t < 30 + len(ILLEGAL[game]):
            a = np.full(n, ILLEGAL[game][t - 30], np.int32)
        else:
            a = deterministic(mask, t)
        acts.append(a)
        outs.append(ref.step(a))
    ref.close()
    data = {k: np.stack([o[k] for o in outs]) for k in outs[0]}
    meta = {"game": game, "case": case, "num_envs": n, "seed": seed, "steps": T}
    path = os.path.join(HERE, f"{game}_{case}.npz")
    np.savez_compressed(path, meta=json.dumps(meta), action=np.stack(acts), **data)
    return path


def main():
    if not hex_othello_lib.ref_available():
        sys.exit("oracle/_ref/libhex_othello_ref.so is missing: run __graft_entry__.build() with an "
                 "envpool checkout")
    for game in hex_othello_lib.GAMES:
        for case in CASES:
            print(record(game, case))


if __name__ == "__main__":
    main()
