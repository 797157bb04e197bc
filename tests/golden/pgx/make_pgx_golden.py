"""Record the PGX TicTacToe-v1 / ConnectFour-v1 fixtures from the reference's own thread pool.

    python tests/golden/pgx/make_pgx_golden.py     # needs oracle/_ref/libpgx_ref.so (build())

Each case is AsyncEnvPool<TicTacToeEnv> / <ConnectFourEnv> (max_num_players 2, one worker
thread, so rows come back in submission order) driven with one action per env (players.env_id =
env_id): a reset, then T steps.  <game>_<case>.npz holds `meta` (JSON: game, num_envs, seed,
steps), `action` [T, n] and every state key as [T + 1, rows, ...] (row 0 of the time axis is the
reset; per-player keys have 2 n rows, the players of env i at 2 i and 2 i + 1).  Cases:
  random      actions over the whole int32 range: in range, -1, the action count, INT_MIN,
              INT_MAX and large values of either sign
  legal       a uniformly random legal action of each env (from the previous mask)
  collide     actions from {0, 1} only: TicTacToe overwrites occupied cells, ConnectFour fills
              columns 0 and 1 and then plays into full columns
  sequence    pgx_deterministic_test.py's sequences (TicTacToe [0, 3, 1, 4, 2], ConnectFour
              [0, 1, 0, 1, 0, 1, 0]) in every env, then the first legal action
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)

from oracle import pgx_lib  # noqa: E402

SEQUENCES = {"TicTacToe": [0, 3, 1, 4, 2], "ConnectFour": [0, 1, 0, 1, 0, 1, 0]}
I32 = np.iinfo(np.int32)


def policy(case, game, rng, t, mask):
    n, A = mask.shape
    if case == "random":
        a = rng.integers(-1, A + 1, size=n)
        special = rng.random(n) < 0.08
        pool = np.array([-1, A, I32.min, I32.max, -(1 << 20), 1 << 20], dtype=np.int64)
        a = np.where(special, pool[rng.integers(0, len(pool), size=n)], a)
        return a.astype(np.int32)
    if case == "legal":
        return np.array([rng.choice(np.flatnonzero(m)) for m in mask], dtype=np.int32)
    if case == "collide":
        return rng.integers(0, 2, size=n).astype(np.int32)
    seq = SEQUENCES[game]
    if t < len(seq):
        return np.full(n, seq[t], dtype=np.int32)
    return np.argmax(mask, axis=1).astype(np.int32)


CASES = {"random": (64, 3, 300), "legal": (64, 5, 300), "collide": (32, 11, 120),
         "sequence": (8, 7, 12)}


def record(game, case):
    n, seed, T = CASES[case]
    rng = np.random.default_rng(seed)
    ref = pgx_lib.PgxRef(game, n, seed=seed)
    outs = [ref.reset()]
    acts = []
    for t in range(T):
        a = policy(case, game, rng, t, outs[-1]["info:legal_action_mask"])
        acts.append(a)
        outs.append(ref.step(a))
    ref.close()
    data = {k: np.stack([o[k] for o in outs]) for k in outs[0]}
    meta = {"game": game, "case": case, "num_envs": n, "seed": seed, "steps": T}
    path = os.path.join(HERE, f"{game}_{case}.npz")
    np.savez_compressed(path, meta=json.dumps(meta), action=np.stack(acts), **data)
    return path


def main():
    if not pgx_lib.ref_available():
        sys.exit("oracle/_ref/libpgx_ref.so is missing: run __graft_entry__.build() with an "
                 "envpool checkout")
    for game in pgx_lib.GAMES:
        for case in CASES:
            print(record(game, case))


if __name__ == "__main__":
    main()
