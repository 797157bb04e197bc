"""Record what the TicTacToe and ConnectFour pools look like from outside into
tests/golden/pgx/pool_layouts.json.

    python tests/golden/pgx/make_pgx_pool_layouts.py   # needs a CUDA device and a built engine

The same record as tests/golden/make_pool_layouts.py keeps for the single-player kinds
(`describe` there: state and action keys with their per-env-row shapes, slab_bytes, the state
blob's size and layout, bytes_per_env_step, the launch count after creation), for every kind in
_capi.TWO_PLAYER_KINDS, both precisions (ignored by these kinds), num_envs 1 and 1000 and iopt
0, -1 and 7 (no iopt is validated).  tests/test_gpu_pgx.py holds every pool to it exactly.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "pool_layouts.json")
sys.path.insert(0, os.path.dirname(HERE))
from make_pool_layouts import describe  # noqa: E402


def cases(kinds):
    for task in kinds:
        for precision in ("f64", "f32"):
            for iopt in (0, -1, 7):
                for n in (1, 1000):
                    yield f"{task}/{precision}/iopt={iopt}/n={n}", (task, precision, iopt, n)


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(HERE))))
    from envpool_b200 import _capi

    out = {name: describe(_capi, *args) for name, args in cases(_capi.TWO_PLAYER_KINDS)}
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {FIXTURE}")


if __name__ == "__main__":
    main()
