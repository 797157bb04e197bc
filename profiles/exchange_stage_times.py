"""Stage times of ONE exchanged step, per rank, un-pipelined (run under torchrun on N GPUs):
CUDA events on the pool's stream around  step(+push)  and  wait  of the direct API
(epb_step_exchange_device / epb_exchange_wait), which serialises  step -> push -> wait  on one
stream.  The first stage is the step kernel and the copy kernel that forwards its rows
(separate launches; the sum is what the events see).  Prints one JSON line per rank: median microseconds of each stage and of the whole step."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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
    st = torch.cuda.ExternalStream(pool.stream, device=dev)
    K = 300
    e = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(K)]
    dist.barrier()
    with torch.cuda.stream(st):
        for k in range(K):
            e[k][0].record(st)
            pool.step_exchange(actions[k % actions.shape[0]])
            e[k][1].record(st)
            pool.exchange_wait()
            e[k][2].record(st)
    pool.sync()
    a = np.array([e[k][0].elapsed_time(e[k][1]) for k in range(50, K)]) * 1e3
    b = np.array([e[k][1].elapsed_time(e[k][2]) for k in range(50, K)]) * 1e3
    tot = e[50][0].elapsed_time(e[K - 1][2]) * 1e3 / (K - 50)
    print(json.dumps({"rank": rank, "world": world, "task": task, "n": n,
                      "step_push_us_med": round(float(np.median(a)), 2),
                      "wait_us_med": round(float(np.median(b)), 2),
                      "step_push_us_p10": round(float(np.percentile(a, 10)), 2),
                      "wait_us_p10": round(float(np.percentile(b, 10)), 2),
                      "whole_step_us": round(tot, 2)}), flush=True)
    dist.barrier()
    pool.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
