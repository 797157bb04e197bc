"""PGX env-step rates on one GPU, next to the reference's CPU thread pool.

    python profiles/pgx_rate.py [--games TicTacToe,ConnectFour] [--out FILE.json]
    python profiles/pgx_rate.py --games Hex,Othello --out profiles/pgx_hex_othello_rate.json

For 65536, 1M and 4M envs of each game, env-steps/s of
  * the captured per-step chain (epb_step_many_timed: CUDA-graph replay of one step launch per
    step, timed between two events inside the graph, steps 16..80 of an 80-step chain) and
  * the fused rollout (epb_rollout_device, 16 steps in one launch, CUDA events around it),
both with uniformly random in-range actions from a [80, n] device stream (most of them illegal
in a busy position, so episodes are short), each the best of 3 repetitions after a warm-up,
with the HBM fraction epb_bytes_per_env_step x rate / 3.35 TB/s (H100 SXM HBM3 data sheet).
A second line drives a legal-random policy on the device: between step_device calls, torch
takes the masked argmax of uniform noise over the last step's info:legal_action_mask, the
pattern of a self-play loop; CUDA events around 64 steps (policy kernels included).  The
reference's own AsyncEnvPool of each game (oracle/_ref) runs on every host
thread at 65536 envs when the build compiled it.  The card's name and power limit are read in
the same run.  Needs a CUDA device: there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
ACTIONS = {"TicTacToe": 9, "ConnectFour": 7, "Hex": 122, "Othello": 65}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def gpu_rates(game, n, torch, CPool):
    pool = CPool(game, n, seed=1)
    rng = np.random.default_rng(0)
    K, m0 = 80, 16
    # rollout steps per launch: 16, fewer where 16 steps of outputs would not fit beside the pool
    T = max(1, min(16, int(40e9 // (n * sum(k.row_bytes for k in pool.keys)))))
    acts = torch.from_numpy(rng.integers(0, ACTIONS[game], size=(K, n)).astype(np.int32)).cuda()
    pool.reset_device()
    chain = []
    for rep in range(4):
        ms = pool.step_many_timed(acts, 0, K, m0, K, use_graph=True)
        if rep:  # the first replay captures the graph
            chain.append((K - m0) * n / (ms * 1e-3))
    tdt = {"int32": torch.int32, "float32": torch.float32, "bool": torch.bool}
    cols = [torch.empty((T, n) + k.shape, dtype=tdt[k.dtype.name], device="cuda")
            for k in pool.keys]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    roll = []
    for rep in range(4):
        torch.cuda.synchronize()
        e0.record()
        pool.rollout_device(acts[:T], T, cols)
        e1.record()
        e1.synchronize()
        if rep:
            roll.append(T * n / (e0.elapsed_time(e1) * 1e-3))
    step_type = cols[[k.name for k in pool.keys].index("step_type")]
    reset_share = float((step_type == 0).double().mean())
    del cols
    # legal-random self-play on the device: masked argmax of uniform noise between steps
    gen = torch.Generator(device="cuda").manual_seed(0)
    pool.reset_device()
    out = pool.outputs_torch()
    mask = out["info:legal_action_mask"]
    legal = []
    for rep in range(4):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(64):
            noise = torch.rand(mask.shape, generator=gen, device="cuda")
            a = torch.where(mask, noise, -1.0).argmax(dim=1).to(torch.int32)
            pool.step_device(a)
        e1.record()
        e1.synchronize()
        if rep:
            legal.append(64 * n / (e0.elapsed_time(e1) * 1e-3))
    done = pool.outputs_torch()["done"]
    b = pool.bytes_per_env_step
    pool.close()
    del acts, out, mask, done
    torch.cuda.empty_cache()
    return {"num_envs": n, "bytes_per_env_step": b, "rollout_T": T,
            "chain_env_steps_per_s": max(chain),
            "chain_hbm_fraction": max(chain) * b / HBM_BYTES_PER_S,
            "rollout_env_steps_per_s": max(roll),
            "rollout_hbm_fraction_at_step_bytes": max(roll) * b / HBM_BYTES_PER_S,
            "rollout_reset_row_share": reset_share,
            "legal_random_step_device_env_steps_per_s": max(legal)}


def ref_rate(game, n):
    from oracle import hex_othello_lib, pgx_lib

    lib, Ref = (hex_othello_lib, hex_othello_lib.HexOthelloRef) if game in hex_othello_lib.GAMES \
        else (pgx_lib, pgx_lib.PgxRef)
    if not lib.ref_available():
        return {"num_envs": n, "env_steps_per_s": "not measured (oracle/_ref was not built)"}
    pool = Ref(game, n, seed=1, num_threads=0)
    acts = np.random.default_rng(0).integers(0, ACTIONS[game], size=(16, n)).astype(np.int32)
    steps = 20
    sec = pool.bench(acts, 5, steps)
    threads = pool.hardware_concurrency()
    pool.close()
    return {"num_envs": n, "env_steps_per_s": steps * n / sec, "host_threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--sizes", default="65536,1048576,4194304")
    ap.add_argument("--games", default="TicTacToe,ConnectFour")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("pgx_rate.py measures the GPU: no CUDA device")
    from envpool_b200._capi import CPool

    games = args.games.split(",")
    res = {"tasks": [f"{g}-v1" for g in games], "card": card(),
           "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S,
           "gpu": {g: [gpu_rates(g, int(n), torch, CPool) for n in args.sizes.split(",")]
                   for g in games},
           "reference_cpu": {g: ref_rate(g, 65536) for g in games},
           "date": time.strftime("%Y-%m-%d")}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
