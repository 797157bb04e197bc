"""PGX Chess / GardnerChess env-step rates on one GPU, next to the reference's CPU thread pool.

    python profiles/chess_rate.py [--out profiles/chess_rate.json]

For 4096, 16384 and 65536 envs of each game, env-steps/s of
  * the captured per-step chain (epb_step_many_timed: CUDA-graph replay of one step launch per
    step, timed between two events inside the graph, steps 16..80 of an 80-step chain) with
    uniformly random in-range labels from a [80, n] device stream (almost all illegal, so most
    steps end a game and the next one resets it), and
  * a legal-random policy on the device, the pattern of a self-play loop: between step_device
    calls torch takes the masked argmax of uniform noise over the last step's
    info:legal_action_mask; CUDA events around 64 steps, policy kernels included,
each the best of 3 repetitions after a warm-up, with epb_bytes_per_env_step (which leaves out the
repetition scan's reads of the stored keys) and the bytes/s it implies.  For the legal-random
loop at 16384 envs, torch.profiler's mean CUDA time of the step kernel is recorded beside the
loop's time per step, and so is the chain's own kernel (launched directly over the same stream)
beside the chain's time per step and the share of its env-steps that generate moves (resets and
legal labels).  The reference's own AsyncEnvPool<ChessEnv> / <GardnerChessEnv>
(oracle/_ref) runs on every host thread at 4096 envs with random in-range labels whose target lies
on the board (it writes board[-1] for the others).  The card's name and power limit are read in
the same run.  Needs a CUDA device: there is no CPU fallback.
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

ACTIONS = {"Chess": 4672, "GardnerChess": 1225}


def gpu_rates(game, n, torch, CPool):
    A = ACTIONS[game]
    pool = CPool(game, n, seed=1)
    rng = np.random.default_rng(0)
    K, m0 = 80, 16
    acts = torch.from_numpy(rng.integers(0, A, size=(K, n)).astype(np.int32)).cuda()
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

    def loop(steps):
        for _ in range(steps):
            noise = torch.rand(mask.shape, generator=gen, device="cuda")
            pool.step_device(torch.where(mask, noise, -1.0).argmax(dim=1).to(torch.int32))

    legal = []
    for rep in range(4):
        torch.cuda.synchronize()
        e0.record()
        loop(64)
        e1.record()
        e1.synchronize()
        if rep:
            legal.append(64 * n / (e0.elapsed_time(e1) * 1e-3))
    out = {"num_envs": n, "bytes_per_env_step": pool.bytes_per_env_step,
           "chain_env_steps_per_s": max(chain),
           "chain_bytes_per_s": max(chain) * pool.bytes_per_env_step,
           "legal_random_step_device_env_steps_per_s": max(legal)}
    if n == 16384:
        from torch.profiler import ProfilerActivity, profile

        def kernel_us(run):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            kern = [e for e in prof.key_averages() if "chess_kernel" in e.key]
            return kern[0].device_time_total / kern[0].count if kern else None

        out["legal_random_step_kernel_us"] = kernel_us(lambda: loop(16))
        out["legal_random_loop_us_per_step"] = 1e6 * n / max(legal)
        # the chain's own kernels: the same random stream, launched directly (not captured)
        pool.reset_device()
        out["chain_step_kernel_us"] = kernel_us(
            lambda: pool.step_many_device(acts, 0, K, use_graph=False))
        out["chain_us_per_step"] = 1e6 * n / max(chain)
        # share of the chain's env-steps that generate moves: resets and legal labels
        pool.reset_device()
        gen = 0
        for k in range(K):
            prev = pool.outputs_torch()
            mask, done = prev["info:legal_action_mask"], prev["done"]
            a = acts[k].long()
            legal = mask.gather(1, a.clamp(0, A - 1)[:, None])[:, 0] & (a >= 0) & (a < A)
            gen += int((done | legal).sum())
            pool.step_device(acts[k])
        out["chain_move_generating_share"] = gen / (K * n)
    pool.close()
    del acts, mask
    torch.cuda.empty_cache()
    return out


def ref_rate(game, n):
    from oracle import chess_lib

    if not chess_lib.ref_available():
        return {"num_envs": n, "env_steps_per_s": "not measured (oracle/_ref was not built)"}
    on_board = np.flatnonzero(chess_lib.ChessOracle(game, 1, obs=False).on_board())
    pool = chess_lib.ChessRef(game, n, seed=1, num_threads=0)
    acts = on_board[np.random.default_rng(0).integers(0, len(on_board), size=(16, n))]
    steps = 20
    sec = pool.bench(acts.astype(np.int32), 5, steps)
    threads = pool.L.pgr_hardware_concurrency()
    pool.close()
    return {"num_envs": n, "env_steps_per_s": steps * n / sec, "host_threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--sizes", default="4096,16384,65536")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("chess_rate.py measures the GPU: no CUDA device")
    from envpool_b200._capi import CPool

    res = {"tasks": [f"{g}-v1" for g in ACTIONS], "card": card(),
           "gpu": {g: [gpu_rates(g, int(n), torch, CPool) for n in args.sizes.split(",")]
                   for g in ACTIONS},
           "reference_cpu": {g: ref_rate(g, 4096) for g in ACTIONS},
           "date": time.strftime("%Y-%m-%d")}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
