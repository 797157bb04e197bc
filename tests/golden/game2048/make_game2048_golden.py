"""Record the Game2048 fixtures in this directory FROM THE REFERENCE ITSELF.

Needs oracle/_ref/libg2048_ref.so compiled from an envpool checkout (`oracle.g2048_lib.build(
<envpool checkout>)`, which `__graft_entry__.build()` runs when it finds one): the reference's
own AsyncEnvPool<Game2048Env> (envpool/jumanji/game2048_env.h), unmodified.

    python tests/golden/game2048/make_game2048_golden.py

The fixtures live in this subdirectory, not beside the other tasks' .npz files, so that the
tests globbing tests/golden/*.npz keep their parameter sets.  Each <name>.npz holds `meta` (json:
seed, max_episode_steps, add_random_cell, initial_board, replay_boards, num_envs), `actions`
[T, N] and one [T+1, N, ...] array per state key (index 0 = the reset() batch, index t+1 = the
batch returned by step(actions[t])).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(
    os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
from oracle.g2048_lib import Game2048Ref  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1

# a board on which no direction moves anything: every reset ends its episode
DEAD_BOARD = "1,2,1,2,2,1,2,1,1,2,1,2,2,1,2,1"
# 3 replay boards (48 cells) of the 32 the config holds: boards 3..31 are all zero
SHORT_REPLAY = ",".join(str(v) for v in
                        [1, 1, 2, 2, 3, 4, 0, 0, 0, 2, 0, 0, 0, 5, 0, 0] +
                        [0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 3] +
                        [6, 5, 4, 3, 5, 4, 3, 2, 4, 3, 2, 1, 3, 2, 1, 1])
START_BOARD = "1,1,2,2,3,4,0,0,0,2,0,0,0,5,0,0"

# name, seed, max_episode_steps, add_random_cell, initial_board, replay_boards, N, T
CASES = [
    ("default", 11, 1000, True, "", "", 64, 1000),
    ("no_random_cell", 12, 1000, False, START_BOARD, "", 32, 200),
    ("dead_initial_board", 13, 1000, True, DEAD_BOARD, "", 8, 40),
    ("short_replay", 14, 1000, True, START_BOARD, SHORT_REPLAY, 32, 300),
    ("max_steps_5", 15, 5, True, "", "", 32, 400),
    ("max_steps_1", 16, 1, True, "", "", 32, 100),
]


def actions_for(rng, T, N):
    """Legal directions mostly; one action in ten is out of range (-5, 4, INT_MIN, INT_MAX),
    which the env clamps to [0, 3]."""
    a = rng.integers(0, 4, size=(T, N)).astype(np.int64)
    odd = rng.random((T, N)) < 0.1
    a[odd] = rng.choice(np.array([-5, 4, INT32_MIN, INT32_MAX]), size=int(odd.sum()))
    return a.astype(np.int32)


def record(name, seed, mes, add_random_cell, initial, replay, N, T):
    rng = np.random.default_rng(seed)
    acts = actions_for(rng, T, N)
    pool = Game2048Ref(N, seed=seed, max_episode_steps=mes, add_random_cell=add_random_cell,
                       initial_board=initial, replay_boards=replay, num_threads=1)
    frames = [pool.reset()]
    for t in range(T):
        frames.append(pool.step(acts[t]))
    pool.close()
    out = {k: np.stack([f[k] for f in frames]) for k in frames[0]}
    meta = dict(task="Game2048", seed=seed, max_episode_steps=mes,
                add_random_cell=add_random_cell, initial_board=initial, replay_boards=replay,
                num_envs=N)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=json.dumps(meta),
                        actions=acts, **out)
    ends = int(out["done"][1:].sum())
    print(f"{name}: {T} steps x {N} envs, {ends} episode ends, highest tile "
          f"{int(out['info:highest_tile'].max())}, trunc {int(out['trunc'].sum())}")


if __name__ == "__main__":
    for case in CASES:
        record(*case)
