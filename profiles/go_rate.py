"""PGX Go env-step rates on one GPU, next to the reference's CPU thread pool.

    python profiles/go_rate.py [--out profiles/go_rate.json]

For 4096 and 65536 envs of each board size (Go9x9, Go13x13, Go19x19), env-steps/s of
  * the captured per-step chain (epb_step_many_timed: CUDA-graph replay of one step launch per
    step, timed between two events inside the graph, steps 16..80 of an 80-step chain) with
    uniformly random in-range actions 0..S^2 from a [80, n] device stream (many of them land on
    occupied cells, so episodes are short), and
  * a legal-random policy on the device, the pattern of a self-play loop: between step_device
    calls torch takes the masked argmax of uniform noise over the last step's
    info:legal_action_mask (the pass only when nothing else is legal, so games run long); CUDA
    events around 64 steps, policy kernels included,
each the best of 3 repetitions after a warm-up, with epb_bytes_per_env_step (which leaves out the
superko scan's reads of the hash history).  The reference's own AsyncEnvPool<GoEnv> (oracle/_ref)
runs on every host thread at 4096 envs with the same random in-range actions when the build
compiled it.  The card's name and power limit are read in the same run.  Needs a CUDA device:
there is no CPU fallback.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "profiles")]

from pgx_rate import card  # noqa: E402

GAMES = {"Go9x9": 9, "Go13x13": 13, "Go19x19": 19}


def gpu_rates(game, n, torch, CPool):
    A = GAMES[game] ** 2
    pool = CPool(game, n, seed=1)
    rng = np.random.default_rng(0)
    K, m0 = 80, 16
    acts = torch.from_numpy(rng.integers(0, A + 1, size=(K, n)).astype(np.int32)).cuda()
    pool.reset_device()
    chain = []
    for rep in range(4):
        ms = pool.step_many_timed(acts, 0, K, m0, K, use_graph=True)
        if rep:  # the first replay captures the graph
            chain.append((K - m0) * n / (ms * 1e-3))
    gen = torch.Generator(device="cuda").manual_seed(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pool.reset_device()
    mask = pool.outputs_torch()["info:legal_action_mask"]
    legal = []
    for rep in range(4):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(64):
            noise = torch.rand(mask.shape, generator=gen, device="cuda")
            noise[:, A] = 0.0  # the pass loses to any other legal move
            a = torch.where(mask, noise, -1.0).argmax(dim=1).to(torch.int32)
            pool.step_device(a)
        e1.record()
        e1.synchronize()
        if rep:
            legal.append(64 * n / (e0.elapsed_time(e1) * 1e-3))
    b = pool.bytes_per_env_step
    pool.close()
    del acts, mask
    torch.cuda.empty_cache()
    return {"num_envs": n, "bytes_per_env_step": b, "chain_env_steps_per_s": max(chain),
            "legal_random_step_device_env_steps_per_s": max(legal)}


def ref_rate(game, n):
    from oracle import go_lib

    if not go_lib.ref_available():
        return {"num_envs": n, "env_steps_per_s": "not measured (oracle/_ref was not built)"}
    pool = go_lib.GoRef(game, n, seed=1, num_threads=0)
    acts = np.random.default_rng(0).integers(0, GAMES[game] ** 2 + 1, size=(16, n)).astype(np.int32)
    steps = 20
    sec = pool.bench(acts, 5, steps)
    threads = pool.hardware_concurrency()
    pool.close()
    return {"num_envs": n, "env_steps_per_s": steps * n / sec, "host_threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--sizes", default="4096,65536")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("go_rate.py measures the GPU: no CUDA device")
    from envpool_b200._capi import CPool

    res = {"tasks": [f"{g}-v1" for g in GAMES], "card": card(),
           "gpu": {g: [gpu_rates(g, int(n), torch, CPool) for n in args.sizes.split(",")]
                   for g in GAMES},
           "reference_cpu": {g: ref_rate(g, 4096) for g in GAMES},
           "date": time.strftime("%Y-%m-%d")}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
