"""Record what every engine pool looks like from outside into pool_layouts.json.

    python tests/golden/make_pool_layouts.py      # needs a CUDA device and a built engine

For every kind in _capi.KINDS, both precisions, num_envs 1 and 1000, and every iopt the kind
accepts plus -1 (the kind's default) and one more value (rejected where the kind validates
iopt), a case holds either the error pool creation raised (class and message) or the state
and action keys, slab_bytes, the state blob's size and its 12 state_layout values,
bytes_per_env_step and the launch count right after creation.  The state blob's layout is
the snapshot format of epb_state_export, so tests/test_gpu_pool_layout.py holds every pool
to these values exactly.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "pool_layouts.json")

# kind -> (the iopt values it accepts, one more value to try)
IOPTS = {
    "CartPole": ([0], 7), "Pendulum": ([0, 1], 7), "Acrobot": ([0], 7),
    "MountainCar": ([0], 7), "MountainCarContinuous": ([0], 7),
    "FrozenLake": ([4, 8], 5), "Catch": ([0], 7), "Taxi": ([0], 7), "NChain": ([0], 7),
    "CliffWalking": ([0, 1], 7), "Blackjack": ([0, 1, 2, 3], 7), "HalfCheetah": ([0], 7),
    "Game2048": ([0, 1], 2), "Minesweeper": ([0], 1),
}


def cases(kinds):
    for task in kinds:
        accepted, other = IOPTS[task]
        for precision in ("f64", "f32"):
            for iopt in accepted + [-1, other]:
                for n in (1, 1000):
                    yield f"{task}/{precision}/iopt={iopt}/n={n}", (task, precision, iopt, n)


def describe(capi, task, precision, iopt, n):
    try:
        pool = capi.CPool(task, n, seed=1, iopt=iopt, precision=precision)
    except Exception as e:  # the error is part of what is pinned
        return {"error": type(e).__name__, "message": str(e)}
    try:
        def key(k):
            return {"name": k.name, "dtype": k.dtype.str, "shape": list(k.shape),
                    "row_bytes": k.row_bytes, "offset": k.offset}

        return {
            "keys": [key(k) for k in pool.keys],
            "action": key(pool.action_key),
            "slab_bytes": pool.slab_bytes,
            "state_bytes": pool.lib.epb_state_bytes(pool.h),
            "state_layout": pool.state_layout(),
            "bytes_per_env_step": pool.bytes_per_env_step,
            "launch_count": pool.launch_count,
        }
    finally:
        pool.close()


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from envpool_b200 import _capi

    out = {name: describe(_capi, *args) for name, args in cases(_capi.KINDS)}
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} cases -> {FIXTURE}")


if __name__ == "__main__":
    main()
