"""Iteration statistics of the HalfCheetah constraint solver on random-action rollouts, from the
host build of the pair-lane kernel source (tests/hc_pair_host/pair_stats.cc, HCP_STATS): how many
merged constraint rows an mj_step has, how many line searches a constrained mj_step needs, how
many passes over the rows a line search needs.  CPU only.

    python profiles/hc_pair_iteration_stats.py [envs] [steps]"""
import ctypes
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from envpool_b200 import _capi

    envs = int(sys.argv[1]) if len(sys.argv) > 1 else 24
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 150
    src = os.path.join(ROOT, "tests", "hc_pair_host", "pair_stats.cc")
    so = os.path.join(ROOT, "tests", "hc_pair_host", "libhc_pair_stats.so")
    subprocess.run(["g++", "-std=c++20", "-O2", "-fPIC", "-shared", "-pthread", "-w", src, "-o", so],
                   check=True)
    H = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    H.hc_pair_host_step.argtypes = [ctypes.c_char_p, vp, vp, vp, vp, ctypes.c_int, ctypes.c_int]
    H.hc_pair_trace.argtypes = [ctypes.c_int, vp, ctypes.c_int]
    blob = _capi.hc_model_blob()
    rng = np.random.default_rng(0)
    for _ in range(envs):   # the env's reset distribution, uniform random actions, frame_skip 5
        q, v, w = rng.uniform(-0.1, 0.1, 9), rng.normal(0, 0.1, 9), np.zeros(9)
        for _ in range(steps):
            a = rng.uniform(-1, 1, 6)
            H.hc_pair_host_step(blob, q.ctypes.data, v.ctypes.data, w.ctypes.data, a.ctypes.data,
                                5, 27)
    nh, lh, rh = np.zeros(32, np.int64), np.zeros(64, np.int64), np.zeros(32, np.int64)
    cap = H.hc_pair_trace(0, None, 0)
    tr = np.zeros(cap, np.int32)
    H.hc_pair_trace(0, tr.ctypes.data, cap)
    newton = passes = 0
    for ev, val in tr.reshape(-1, 2):                 # event codes: mujoco_pair.cuh, TR_*
        if ev == 1:                                   # a constraint solve starts
            rh[min(val, 31)] += 1
        elif ev == 3:                                 # a Newton step's line search
            newton += 1
            passes = 0
            if val != 0:                              # skipped: no row pass
                lh[0] += 1
        elif ev == 4:                                 # an update of alpha, after a row pass
            passes += 1
        elif ev == 5:                                 # ended; converged or stalled on a pass
            lh[min(passes + (val != 2), 63)] += 1
        elif ev == 6:                                 # the Newton loop ends
            nh[min(newton, 31)] += 1
            newton = 0
    print("merged constraint rows per mj_step:", {i: int(x) for i, x in enumerate(rh) if x},
          f"-> {100 * rh[0] / rh.sum():.0f} % of the mj_steps have none")
    print("line searches per constrained mj_step:", {i: int(x) for i, x in enumerate(nh) if x},
          f"mean {(nh * np.arange(32)).sum() / max(nh.sum(), 1):.2f}")
    print("row passes per line search (the first is fused with the J*search pass):",
          {i: int(x) for i, x in enumerate(lh) if x},
          f"mean {(lh * np.arange(64)).sum() / max(lh.sum(), 1):.2f}")


if __name__ == "__main__":
    main()
