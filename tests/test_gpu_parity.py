"""GPU parity tests: the CUDA engine, driven through the C ABI, against
  (1) the golden trajectories recorded from the reference itself (tests/golden),
  (2) the CPU restatement oracle (oracle/ep_oracle.c) on seeded random rollouts,
  (3) size-independent properties at BASELINE.json's full sizes.
Bar: integer / bool / index columns bit-exact.  Float columns: the f64 engine mode is
required to match within FLOAT_ATOL_F64 (CUDA's sin/cos differ from glibc's by <= 2 ulp in
double, which can flip the last bit of a float32 output); the f32 mode within 2e-5 per
teacher-forced step and 1e-3 over a short free-running horizon.
"""
import numpy as np
import pytest

from helpers import (REGISTERED, assert_batch_equal, golden_cases, load_golden,
                     random_actions)

pytestmark = pytest.mark.gpu

FLOAT_ATOL_F64 = 1e-6   # relative-absolute: |err| <= atol * (1 + |ref|)

CLASSIC = ["CartPole", "Pendulum", "Acrobot", "MountainCar", "MountainCarContinuous"]
TOY = ["FrozenLake", "Catch", "Taxi", "NChain", "CliffWalking", "Blackjack"]


@pytest.mark.parametrize("case", golden_cases())
def test_golden_trajectories_host_path(capi, case):
    meta, gold = load_golden(case)
    pool = capi.CPool(meta["task"], meta["num_envs"], seed=meta["seed"],
                      max_episode_steps=meta["max_episode_steps"], iopt=meta["iopt"])
    acts = gold["actions"]
    keys = [k for k in gold if k != "actions"]
    got = pool.reset()
    assert_batch_equal(got, {k: gold[k][0] for k in keys}, meta["task"], FLOAT_ATOL_F64,
                       f"{case} reset")
    for t in range(acts.shape[0]):
        got = pool.step(acts[t])
        assert_batch_equal(got, {k: gold[k][t + 1] for k in keys}, meta["task"],
                           FLOAT_ATOL_F64, f"{case} t={t}")
    pool.close()


@pytest.mark.parametrize("task", CLASSIC + TOY)
def test_oracle_random_rollout(capi, task):
    from oracle.oracle_lib import OraclePool

    ms, iopt = REGISTERED[task]
    N, T = 2048, 300
    rng = np.random.default_rng(123)
    pool = capi.CPool(task, N, seed=11, max_episode_steps=ms, iopt=iopt)
    orc = OraclePool(task, N, seed=11, max_episode_steps=ms, iopt=iopt)
    assert_batch_equal(pool.reset(), orc.reset(), task, FLOAT_ATOL_F64, f"{task} reset")
    for t in range(T):
        a = random_actions(task, rng, (N,))
        assert_batch_equal(pool.step(a), orc.step(a), task, FLOAT_ATOL_F64, f"{task} t={t}")
    pool.close()


@pytest.mark.parametrize("task,iopt,ms", [("FrozenLake", 8, 200), ("CliffWalking", 1, -1),
                                          ("Blackjack", 1, -1), ("Blackjack", 0, -1),
                                          ("Pendulum", 0, 200)])
def test_oracle_option_variants(capi, task, iopt, ms):
    from oracle.oracle_lib import OraclePool

    N, T = 1024, 250
    rng = np.random.default_rng(5)
    pool = capi.CPool(task, N, seed=3, max_episode_steps=ms, iopt=iopt)
    orc = OraclePool(task, N, seed=3, max_episode_steps=ms, iopt=iopt)
    assert_batch_equal(pool.reset(), orc.reset(), task, FLOAT_ATOL_F64, "reset")
    for t in range(T):
        a = random_actions(task, rng, (N,))
        assert_batch_equal(pool.step(a), orc.step(a), task, FLOAT_ATOL_F64, f"t={t}")


@pytest.mark.parametrize("precision,atol", [("f64", FLOAT_ATOL_F64), ("f32", 2e-5)])
@pytest.mark.parametrize("task", CLASSIC)
def test_teacher_forced_single_step(capi, task, precision, atol):
    """Per-step arithmetic parity without chaotic amplification: before every step the
    oracle is overwritten with the engine's own state (exported through
    epb_state_export), then both advance one step on the same action.  f64 mode must agree
    to FLOAT_ATOL_F64, f32 mode to 2e-5 (relative-absolute).  A threshold event may
    straddle in f32 (done one step early/late); such an env is dropped from then on, and the
    drop rate is bounded."""
    from oracle.oracle_lib import OraclePool

    ms, iopt = REGISTERED[task]
    N, T = 384, 140
    rng = np.random.default_rng(17)
    pool = capi.CPool(task, N, seed=6, max_episode_steps=ms, iopt=iopt, precision=precision)
    orc = OraclePool(task, N, seed=6, max_episode_steps=ms, iopt=iopt)
    g, w = pool.reset(), orc.reset()
    alive = np.ones(N, dtype=bool)
    for t in range(T):
        st = pool.state_arrays(pool.state_export())
        rs = st["rstate"].astype(np.float64)
        for e in range(N):
            s5 = list(rs[:, e]) + [0.0] * (5 - rs.shape[0])
            orc.set_state(e, s5, int(st["flags"][e] & 1), int(st["flags"][e] >> 1))
        a = random_actions(task, rng, (N,))
        g, w = pool.step(a), orc.step(a)
        flags_ok = (g["done"] == w["done"]) & (g["elapsed_step"] == w["elapsed_step"]) & \
                   (g["trunc"] == w["trunc"])
        if precision == "f64":
            assert flags_ok.all(), (task, t, np.argwhere(~flags_ok)[:5])
        alive &= flags_ok
        for k in ("obs", "reward", "info:state"):
            if k not in w:
                continue
            err = np.abs(g[k].astype(np.float64) - w[k]) / (1 + np.abs(w[k]))
            assert err[alive].max() <= atol, (task, precision, t, k, float(err[alive].max()))
    assert alive.mean() >= 0.97, alive.mean()


@pytest.mark.parametrize("task", CLASSIC)
def test_f32_mode_free_running_short_horizon(capi, task):
    """f32 engine mode against the double oracle, free running for 25 steps from the same
    reset: stated tolerance 1e-3 (relative-absolute) while an env's flags still agree."""
    from oracle.oracle_lib import OraclePool

    ms, iopt = REGISTERED[task]
    N, T = 4096, 25
    rng = np.random.default_rng(9)
    pool = capi.CPool(task, N, seed=21, max_episode_steps=ms, iopt=iopt, precision="f32")
    orc = OraclePool(task, N, seed=21, max_episode_steps=ms, iopt=iopt)
    g, w = pool.reset(), orc.reset()
    in_sync = np.ones(N, dtype=bool)
    for t in range(T):
        a = random_actions(task, rng, (N,))
        g, w = pool.step(a), orc.step(a)
        in_sync &= (g["done"] == w["done"]) & (g["elapsed_step"] == w["elapsed_step"])
        err = np.abs(g["obs"].astype(np.float64) - w["obs"]) / (1 + np.abs(w["obs"]))
        assert err[in_sync].max() <= 1e-3, (task, t, float(err[in_sync].max()))
    assert in_sync.mean() >= 0.98, in_sync.mean()


@pytest.mark.parametrize("task", ["CartPole", "FrozenLake", "Catch", "Blackjack", "Acrobot",
                                  "Taxi", "NChain", "CliffWalking", "CliffWalking-slippery"])
def test_device_path_and_rollout_match_host_path(capi, task):
    import torch

    task, _, slippery = task.partition("-")
    ms, iopt = REGISTERED[task]
    iopt = 1 if slippery else iopt
    N, T = 3000, 40   # not a multiple of the CTA size: exercises the tail CTA
    rng = np.random.default_rng(2)
    acts = random_actions(task, rng, (T, N))
    host = capi.CPool(task, N, seed=5, max_episode_steps=ms, iopt=iopt)
    dev = capi.CPool(task, N, seed=5, max_episode_steps=ms, iopt=iopt)
    roll = capi.CPool(task, N, seed=5, max_episode_steps=ms, iopt=iopt)
    ref = [host.reset()] + [host.step(acts[t]) for t in range(T)]
    # device-resident single steps
    d_acts = torch.from_numpy(acts).cuda()
    dev.reset_device()
    dev.sync()
    got = {k: v.cpu().numpy() for k, v in dev.outputs_torch().items()}
    assert_batch_equal(got, ref[0], task, 0.0, "device reset")
    for t in range(T):
        dev.step_device(d_acts[t])
        dev.sync()
        got = {k: v.cpu().numpy() for k, v in dev.outputs_torch().items()}
        assert_batch_equal(got, ref[t + 1], task, 0.0, f"device t={t}")
    # fused rollout: one launch for all T steps
    roll.reset_device()
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((T, N) + k.shape, dtype=tdt[k.dtype], device="cuda")
            for k in roll.keys]
    roll.rollout_device(d_acts, T, cols)
    roll.sync()
    for t in range(T):
        got = {k.name: c[t].cpu().numpy() for k, c in zip(roll.keys, cols)}
        assert_batch_equal(got, ref[t + 1], task, 0.0, f"rollout t={t}")


@pytest.mark.parametrize("task", ["CartPole", "Taxi"])
def test_env_id_routing_and_partial_reset(capi, task):
    """Sync-mode row i <-> env env_id[i] (state_buffer.h:94-97); partial-id reset/step."""
    from oracle.oracle_lib import OraclePool

    ms, iopt = REGISTERED[task]
    N = 512
    rng = np.random.default_rng(4)
    pool = capi.CPool(task, N, seed=1, max_episode_steps=ms, iopt=iopt)
    orc = OraclePool(task, N, seed=1, max_episode_steps=ms, iopt=iopt)
    assert_batch_equal(pool.reset(), orc.reset(), task, FLOAT_ATOL_F64, "reset")
    for t in range(30):
        perm = rng.permutation(N).astype(np.int32)
        a = random_actions(task, rng, (N,))
        assert_batch_equal(pool.step(a, perm), orc.step(a, perm), task, FLOAT_ATOL_F64,
                           f"perm t={t}")
    sub = rng.choice(N, size=100, replace=False).astype(np.int32)
    assert_batch_equal(pool.reset(sub), orc.reset(sub), task, FLOAT_ATOL_F64, "partial reset")
    a = random_actions(task, rng, (100,))
    assert_batch_equal(pool.step(a, sub), orc.step(a, sub), task, FLOAT_ATOL_F64,
                       "partial step")


def test_env_seed_list_and_errors(capi):
    from oracle.oracle_lib import OraclePool

    seeds = np.arange(100, 164, dtype=np.int32)[::-1].copy()
    pool = capi.CPool("CartPole", 64, env_seed=seeds, max_episode_steps=500)
    orc = OraclePool("CartPole", 64, env_seed=seeds, max_episode_steps=500)
    assert_batch_equal(pool.reset(), orc.reset(), "CartPole", FLOAT_ATOL_F64, "env_seed")
    with pytest.raises(ValueError):
        capi.CPool("CartPole", 8, batch_size=9)          # env_spec.h:75-80
    with pytest.raises(ValueError):
        pool.step(np.zeros(64, np.int32), np.full(64, 64, np.int32))  # id out of range
    with pytest.raises(capi.EpbError):
        pool.recv()                                       # nothing outstanding


@pytest.mark.parametrize("task", ["FrozenLake", "CartPole", "Pendulum", "Catch", "Taxi", "NChain",
                                  "CliffWalking", "Blackjack"])
def test_snapshot_roundtrip(capi, task):
    """The state blob is the whole env state (classic_control: the reset-ahead records
    travel with it)."""
    N = 1000
    ms, iopt = REGISTERED[task]
    ms = min(ms, 30)   # several resets inside the compared window
    rng = np.random.default_rng(8)
    a = capi.CPool(task, N, seed=2, max_episode_steps=ms, iopt=iopt)
    a.reset()
    for _ in range(20):
        a.step(random_actions(task, rng, (N,)))
    blob = a.state_export()
    acts = random_actions(task, rng, (45, N))
    want = [a.step(acts[t]) for t in range(45)]
    b = capi.CPool(task, N, seed=999, max_episode_steps=ms, iopt=iopt)
    b.state_import(blob)
    for t in range(45):
        assert_batch_equal(b.step(acts[t]), want[t], task, 0.0, f"snapshot t={t}")


# ---- BASELINE.json full sizes: size-independent properties -------------------------------
FULL = [("CartPole", 65536), ("Pendulum", 1 << 20), ("Acrobot", 1 << 20),
        ("FrozenLake", 1 << 22), ("Catch", 1 << 22)]


@pytest.mark.parametrize("task,N", FULL)
def test_full_size_properties(capi, task, N):
    """At BASELINE sizes: (a) env-id sharding invariance -- two half pools with
    env_id_offset reproduce the full pool bit-for-bit (the multi-GPU partition, SURVEY 8e);
    (b) a prefix of envs matches the CPU oracle exactly; (c) column invariants."""
    import torch
    from oracle.oracle_lib import OraclePool

    ms, iopt = REGISTERED[task]
    T = 12 if N > (1 << 20) else 25
    P = 4096
    rng = np.random.default_rng(77)
    full = capi.CPool(task, N, seed=0, max_episode_steps=ms, iopt=iopt)
    lo = capi.CPool(task, N // 2, seed=0, max_episode_steps=ms, iopt=iopt)
    hi = capi.CPool(task, N // 2, seed=0, max_episode_steps=ms, iopt=iopt,
                    env_id_offset=N // 2)
    orc = OraclePool(task, P, seed=0, max_episode_steps=ms, iopt=iopt)
    pools = (full, lo, hi)
    for p in pools:
        p.reset_device()
    w = orc.reset()
    for t in range(T + 1):
        for p in pools:
            p.sync()
        f = full.outputs_torch()
        l, h = lo.outputs_torch(), hi.outputs_torch()
        for k in f:
            assert torch.equal(f[k][: N // 2], l[k]), (task, t, k, "lo shard")
            assert torch.equal(f[k][N // 2:], h[k]), (task, t, k, "hi shard")
        got = {k: v[:P].cpu().numpy() for k, v in f.items()}
        assert_batch_equal(got, w, task, FLOAT_ATOL_F64, f"{task} full t={t}")
        assert torch.equal(f["info:env_id"], torch.arange(N, device="cuda", dtype=torch.int32))
        assert bool(((f["discount"] == 0) == f["done"]).all())
        assert bool((f["trunc"] <= f["done"]).all())
        if t == T:
            break
        a = random_actions(task, rng, (N,))
        d_a = torch.from_numpy(a).cuda()
        full.step_device(d_a)
        lo.step_device(d_a[: N // 2].contiguous())
        hi.step_device(d_a[N // 2:].contiguous())
        w = orc.step(a[:P])
