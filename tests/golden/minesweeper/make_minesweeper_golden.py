"""Record the Minesweeper fixtures in this directory FROM THE REFERENCE ITSELF.

Needs oracle/_ref/libms_ref.so compiled from an envpool checkout (`oracle.ms_lib.build(<envpool
checkout>)`, which `__graft_entry__.build()` runs when it finds one): the reference's own
AsyncEnvPool<MinesweeperEnv> (envpool/jumanji/minesweeper_env.h), unmodified.

    python tests/golden/minesweeper/make_minesweeper_golden.py

Each <name>.npz holds `meta` (json: seed, max_episode_steps, the four config strings,
num_envs), `actions` [T, N, 2] and one [T+1, N, ...] array per state key (index 0 = the reset()
batch, index t+1 = the batch returned by step(actions[t])).
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(
    os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
from oracle.ms_lib import MinesweeperRef  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1

# duplicates (5, 17) and out-of-range entries (-3, 100, 250) are dropped: mines {0, 5, 17, 33, 99}
MINES = "5,5,17,-3,100,250,33,0,99,17"
# every location out of range: random placement of 10 mines, as for an empty string
MINES_OUT_OF_RANGE = "-1,100,1000"
# 3 replay boards (300 cells) of the 32 the config holds: boards 3..31 are all -1
REPLAY = ",".join(str(v) for v in np.random.default_rng(2026).integers(-1, 9, size=300))
REWARDS = "0.5,-2.25,7,0.125"
# no token reads as true ("1" | "True" | "true"): 32 replay steps, then the env plays
DONE_NONE = "0,False,,yes"
DONE_AT_2 = "0,True"

# name, seed, max_episode_steps, mine_locations, replay_boards, replay_rewards, replay_done, N, T
CASES = [
    ("default", 11, 90, "", "", "", "", 64, 200),
    ("configured_mines", 12, 90, MINES, "", "", "", 32, 200),
    ("mines_out_of_range", 13, 90, MINES_OUT_OF_RANGE, "", "", "", 32, 200),
    ("short_replay", 14, 90, "", REPLAY, REWARDS, DONE_NONE, 16, 120),
    ("replay_done", 15, 90, MINES, REPLAY, REWARDS, DONE_AT_2, 16, 60),
    ("max_steps_5", 16, 5, "", "", "", "", 32, 200),
    ("max_steps_1", 17, 1, "", "", "", "", 32, 100),
]


def actions_for(rng, T, N):
    """(row, column) uniform in [0, 9]; one component in ten out of range (-5, 10, INT_MIN,
    INT_MAX), which the env clamps to [0, 9]."""
    a = rng.integers(0, 10, size=(T, N, 2)).astype(np.int64)
    odd = rng.random((T, N, 2)) < 0.1
    a[odd] = rng.choice(np.array([-5, 10, INT32_MIN, INT32_MAX]), size=int(odd.sum()))
    return a.astype(np.int32)


def record(name, seed, mes, mines, replay, rewards, done, N, T):
    rng = np.random.default_rng(seed)
    acts = actions_for(rng, T, N)
    pool = MinesweeperRef(N, seed=seed, max_episode_steps=mes, mine_locations=mines,
                          replay_boards=replay, replay_rewards=rewards, replay_done=done,
                          num_threads=1)
    frames = [pool.reset()]
    for t in range(T):
        frames.append(pool.step(acts[t]))
    pool.close()
    out = {k: np.stack([f[k] for f in frames]) for k in frames[0]}
    meta = dict(task="Minesweeper", seed=seed, max_episode_steps=mes, mine_locations=mines,
                replay_boards=replay, replay_rewards=rewards, replay_done=done, num_envs=N)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=json.dumps(meta),
                        actions=acts, **out)
    ends = int(out["done"][1:].sum())
    print(f"{name}: {T} steps x {N} envs, {ends} episode ends, trunc {int(out['trunc'].sum())}, "
          f"solved {int((out['done'][1:] & (out['reward'][1:] == 1)).sum())}")


if __name__ == "__main__":
    for case in CASES:
        record(*case)
