"""Minesweeper-v0 env-step rate on one GPU, next to the reference's CPU thread pool.

    python profiles/minesweeper_rate.py [--out FILE.json]

For 65536, 1M and 4M envs (default config: 10 random mines, no replay, uniformly random
(row, column) clicks): env-steps/s of
  * the captured per-step chain (epb_step_many_timed: CUDA-graph replay of one step launch per
    step, timed between two events inside the graph, steps 16..80 of an 80-step chain), and
  * the fused rollout (epb_rollout_device, 16 steps in one launch, CUDA events around it; 16
    because its output columns hold 534 B per env-step: 36 GB at 4M envs),
each the best of 3 repetitions after a warm-up, with the HBM fraction: epb_bytes_per_env_step
(algorithmic bytes of the single-step kernel) x rate / 3.35 TB/s (H100 SXM HBM3 data sheet).
The rollout keeps env state in registers, so its bytes per step are fewer than the step
kernel's; its fraction is stated against the same per-step bytes and says how fast it is, not
how busy HBM is.  epb_bytes_per_env_step leaves out the 50 mt19937 words of each reset, so the
rollout's rows also give the share of reset rows (step_type 0) and the mean episode length in
steps (reset rows excluded) under this policy.  The reference's own
AsyncEnvPool<MinesweeperEnv> (oracle/_ref) is timed on the host CPU at 65536 envs when the build
compiled it.  The card's name and power limit are read
in the same run.  Needs a CUDA device: there is no CPU fallback.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def gpu_rates(n, torch, CPool):
    pool = CPool("Minesweeper", n, seed=1, max_episode_steps=90)
    rng = np.random.default_rng(0)
    K, m0, T = 80, 16, 16
    acts = torch.from_numpy(rng.integers(0, 10, size=(K, n, 2)).astype(np.int32)).cuda()
    pool.reset_device()
    chain = []
    for rep in range(4):
        ms = pool.step_many_timed(acts, 0, K, m0, K, use_graph=True)
        if rep:  # the first replay captures the graph
            chain.append((K - m0) * n / (ms * 1e-3))
    cols = [torch.empty((T, n) + k.shape, dtype={"int32": torch.int32, "float32": torch.float32,
                                                 "bool": torch.bool}[k.dtype.name],
                        device="cuda") for k in pool.keys]
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
    b = pool.bytes_per_env_step
    pool.close()
    del cols, acts
    torch.cuda.empty_cache()
    return {"num_envs": n, "bytes_per_env_step": b,
            "chain_env_steps_per_s": max(chain), "chain_hbm_fraction": max(chain) * b / HBM_BYTES_PER_S,
            "rollout_env_steps_per_s": max(roll),
            "rollout_hbm_fraction_at_step_bytes": max(roll) * b / HBM_BYTES_PER_S,
            "rollout_reset_row_share": reset_share,
            "mean_episode_steps": 1.0 / reset_share - 1.0}


def ref_rate(n):
    from oracle import ms_lib

    if not ms_lib.ref_available():
        return {"num_envs": n, "env_steps_per_s": "not measured (oracle/_ref was not built)"}
    pool = ms_lib.MinesweeperRef(n, seed=1, max_episode_steps=90, num_threads=0)
    acts = np.random.default_rng(0).integers(0, 10, size=(16, n, 2)).astype(np.int32)
    steps = 20
    sec = pool.bench(acts, 5, steps)
    threads = pool.hardware_concurrency()
    pool.close()
    return {"num_envs": n, "env_steps_per_s": steps * n / sec, "host_threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--sizes", default="65536,1048576,4194304")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("minesweeper_rate.py measures the GPU: no CUDA device")
    from envpool_b200._capi import CPool

    res = {"task": "Minesweeper-v0", "card": card(), "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S,
           "gpu": [gpu_rates(int(n), torch, CPool) for n in args.sizes.split(",")],
           "reference_cpu": ref_rate(65536),
           "date": time.strftime("%Y-%m-%d")}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
