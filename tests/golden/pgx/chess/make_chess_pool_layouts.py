"""Record what the Chess pools look like from outside into tests/golden/pgx/chess/pool_layouts.json.

    python tests/golden/pgx/chess/make_chess_pool_layouts.py   # needs a CUDA device

The record of ../make_pgx_pool_layouts.py (`describe` of tests/golden/make_pool_layouts.py over
the same precisions, iopts and num_envs) for every kind in _capi.CHESS_KINDS.
tests/test_gpu_pgx_chess.py holds every pool to it exactly.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "pool_layouts.json")
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
from make_pgx_pool_layouts import cases  # noqa: E402
from make_pool_layouts import describe  # noqa: E402


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(HERE)))))
    from envpool_b200 import _capi

    out = {name: describe(_capi, *args) for name, args in cases(_capi.CHESS_KINDS)}
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {FIXTURE}")


if __name__ == "__main__":
    main()
