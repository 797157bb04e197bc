"""Timeline of a captured exchange chain (torchrun, N GPUs, ENVPOOL_B200_EXCHANGE_TRACE=1): per
exchanged step, when the push kernel started / had its credit / published and when the wait kernel
started / saw the last peer flag / ended, in microseconds relative to the first stamp shown."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["ENVPOOL_B200_EXCHANGE_TRACE"] = "1"
import bench  # noqa: E402


def main():
    import torch
    import torch.distributed as dist

    from envpool_b200 import _capi

    task = sys.argv[1] if len(sys.argv) > 1 else "CartPole-v1"
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    eng, ms, iopt, _ = bench.TASKS[task]
    pool = _capi.CPool(eng, n, seed=0, max_episode_steps=ms, iopt=iopt, device=local,
                       env_id_offset=rank * n)
    actions = bench.make_action_stream(torch, task, n, dev, 2 * bench.L2_BYTES)
    err = bench.attach_exchange(torch, dist, pool, world, rank, dev)
    assert not err, err
    pool.step_exchange(None)
    pool.exchange_wait()
    pool.sync()
    K, lead = 24, 40
    for rep in range(3):      # the last replay is the one read back
        dist.barrier()
        ms_ = pool.step_many_timed(actions, 0, lead + K, lead, lead + K, True, True)
    first = 1 + 2 * (lead + K) + lead       # exchanged steps before the timed window of replay 3
    tr = pool.exchange_trace(first + K).astype(np.float64)[first:first + K, :8]
    t0 = tr[tr > 0].min()
    rel = np.where(tr > 0, (tr - t0) / 1e3, -1.0)
    print(json.dumps({"rank": rank, "task": task, "n": n, "us_per_step": round(ms_ / K * 1e3, 2),
                      "depth": os.environ.get("ENVPOOL_B200_EXCHANGE_DEPTH", "4"),
                      "push_ctas": os.environ.get("ENVPOOL_B200_PUSH_CTAS", "default"),
                      "cols": ["push_start", "push_credit", "push_publish", "wait_start",
                               "wait_flag", "wait_end", "push_cta0_stored", "push_cta0_fenced"],
                      "rows_us": [[round(float(v), 1) for v in r] for r in rel]}), flush=True)
    dist.barrier()
    pool.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
