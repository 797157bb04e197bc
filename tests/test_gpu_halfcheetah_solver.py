"""GPU: hc_pair_kernel's constraint solver on the crafted states of tests/hc_solver_cases.py, which
drive the solver of the kernel's source through every branch it can reach (the CPU suite,
test_hc_solver_branches.py, shows which on the host build).

With frame_skip 1 a step is one mj_step, and the qacc_warmstart the kernel writes back
(rstate[18:27]) is exactly its solver's answer.  That answer is held to the extended-precision
minimiser of the problem (scale * (cost - cost*) <= 1e-8 everywhere, scale * |grad| <= 1e-8 where
the solver stopped on the gradient test; on the extreme family, where the line search runs on
rounding noise, the device may stop elsewhere than the host build, so only the gap), and the
state after the step to the oracle at bars tighter than the 1e-9 of the other HalfCheetah tests.
With frame_skip 5 the env steps are teacher-forced against the oracle.  Launch shapes: a small
pool (27 rows per lane in shared memory), 32768 and 32761 envs (the benchmark's 10, the last CTA
partial), and a forced budget of 9 in a subprocess.  Entry points: host step, step_device, a
captured chain, rollout_device over T > 1; they agree bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

import hc_solver_cases as hc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.gpu

FORCE = "ENVPOOL_B200_HC_PAIR_KS"
RESOLVED_BAR = 2e-11   # device vs oracle after one mj_step, relative-absolute
EXTREME_BAR = 2e-10
FS5_BAR = 1e-10        # per teacher-forced env step of 5 mj_steps (resolved states)


@pytest.fixture(scope="module")
def crafted():
    c = hc.cases()
    exits = [hc.parse(hc.host_step(s, a)[1])[0]["exit"] for s, a in zip(c["states"], c["ctrl"])]
    return dict(c, exits=exits)


@pytest.fixture(scope="module")
def oracle():
    return hc.Oracle()


def place(pool, states, envs):
    blob = pool.state_export()
    rs = pool.state_arrays(blob)["rstate"]
    rs[:27, envs] = states[np.arange(len(envs)) % len(states)].T
    return blob


def actions(crafted, n, envs):
    a = np.zeros((n, 6))
    a[envs] = crafted["ctrl"][np.arange(len(envs)) % len(crafted["ctrl"])]
    return a


def check_one_mj_step(crafted, oracle, after, envs, ctx):
    """after: rstate [NR, n] (its first 27 rows: qpos, qvel, qacc_warmstart) after one frame_skip-1 step from the crafted states placed in envs
    (state i % len(states) in envs[i]).  Asserts the bars; returns the worst error against the
    oracle per family class and {branch: (worst gap, worst grad)}."""
    from test_hc_solver_branches import solver_gaps

    k = len(crafted["states"])
    idx = np.arange(len(envs)) % k
    got = after[:27, envs].T
    errs = {"resolved": 0.0, "extreme": 0.0}
    for j, i in enumerate(idx):
        want, _ = oracle.step(crafted["states"][i], crafted["ctrl"][i])
        e = float(np.max(np.abs(got[j] - want) / (1 + np.abs(want))))
        key = "extreme" if crafted["family"][i] == "extreme" else "resolved"
        errs[key] = max(errs[key], e)
        bar = EXTREME_BAR if key == "extreme" else RESOLVED_BAR
        assert e <= bar, (ctx, j, crafted["family"][i], e)
    # the first len(states) placed envs carry every crafted state once
    exits = [x if f != "extreme" else None for x, f in zip(crafted["exits"], crafted["family"])]
    res = solver_gaps(crafted["states"], crafted["ctrl"], crafted["family"], got[:k, 18:27], exits,
                      oracle)
    per = {}
    for r, h in zip(res, crafted["hits"]):
        if r is None:
            continue
        for b in h:
            g, n = per.get(b, (0.0, 0.0))
            per[b] = (max(g, r[0]), max(n, r[1] or 0.0))
    return errs, per


def print_table(ctx, errs, per):
    print(f"\n{ctx}: worst rel err vs oracle {errs}")
    for b, _ in hc.BRANCHES:
        if b in per:
            print(f"  {b:14s} worst gap {per[b][0]:.1e}  worst grad {per[b][1]:.1e}")


def test_small_pool_against_the_minimiser(capi, crafted, oracle):
    k = len(crafted["states"])
    n = 2 * k + 5
    pool = capi.CPool("HalfCheetah", n, seed=2, max_episode_steps=1000, frame_skip=1)
    if FORCE not in os.environ:
        assert pool.hc_pair_rows() == 27
    pool.reset()
    envs = np.arange(2 * k)
    pool.state_import(place(pool, crafted["states"], envs))
    pool.step(actions(crafted, n, envs))
    after = pool.state_arrays(pool.state_export())["rstate"]
    errs, per = check_one_mj_step(crafted, oracle, after, envs, "small pool")
    print_table(f"{n} envs, ks={pool.hc_pair_rows()}", errs, per)


def test_frame_skip_5_teacher_forced(capi, crafted):
    from oracle.oracle_lib import OraclePool

    k = len(crafted["states"])
    n = k
    pool = capi.CPool("HalfCheetah", n, seed=2, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=2, max_episode_steps=1000)
    pool.reset(), orc.reset()
    envs = np.arange(k)
    pool.state_import(place(pool, crafted["states"], envs))
    resolved = np.array([f != "extreme" for f in crafted["family"]])
    worst = 0.0
    rng = np.random.default_rng(4)
    for t in range(4):
        st = pool.state_arrays(pool.state_export())
        for e in range(n):
            orc.mjc_set(e, st["rstate"][:27, e], int(st["flags"][e] & 1), int(st["flags"][e] >> 1))
        a = actions(crafted, n, envs) if t == 0 else rng.uniform(-1.5, 1.5, (n, 6))
        pool.step(a), orc.step(a)
        g = pool.state_arrays(pool.state_export())["rstate"][:27].T
        w = np.array([orc.mjc_get(e) for e in range(n)])
        err = np.max(np.abs(g - w) / (1 + np.abs(w)), axis=1)
        assert err[resolved].max() <= FS5_BAR, (t, err[resolved].max())
        worst = max(worst, float(err[resolved].max()))
    # the extreme family is not held here: over 5 mj_steps its noise-driven solver paths diverge
    print(f"\nframe_skip 5, teacher-forced: worst rel err vs oracle {worst:.2e} (resolved states)")


@pytest.mark.parametrize("n", [32768, 32761])
def test_benchmark_shape_through_every_entry_point(capi, crafted, oracle, n):
    import torch

    if FORCE in os.environ:
        pytest.skip(f"{FORCE} is set")
    K = 3
    rng = np.random.default_rng(n)
    k = len(crafted["states"])
    envs = np.union1d(np.r_[0:k, n - 33:n], rng.choice(n, 100, replace=False))
    envs = np.r_[np.arange(k), np.setdiff1d(envs, np.arange(k))]
    names = ("step", "step_device", "graph", "rollout")
    pools = {m: capi.CPool("HalfCheetah", n, seed=11, max_episode_steps=1000, frame_skip=1)
             for m in names}
    pools["step"].reset()
    blob = place(pools["step"], crafted["states"], envs)
    for p in pools.values():
        p.state_import(blob)
    acts = np.stack([actions(crafted, n, envs)] + [rng.uniform(-1.5, 1.5, (n, 6))
                                                   for _ in range(K - 1)])
    d_acts = torch.from_numpy(acts).cuda()
    host = []
    for t in range(K):
        host.append(pools["step"].step(acts[t]))
        if t == 0:
            after = pools["step"].state_arrays(pools["step"].state_export())["rstate"]
            errs, per = check_one_mj_step(crafted, oracle, after, envs, f"n={n}")
            print_table(f"{n} envs, ks={pools['step'].hc_pair_rows()}", errs, per)

    def outputs(p):
        p.sync()
        return {kk: v.cpu().numpy() for kk, v in p.outputs_torch().items()}

    for t in range(K):
        pools["step_device"].step_device(d_acts[t])
        o = outputs(pools["step_device"])
        assert all(o[kk].tobytes() == host[t][kk].tobytes() for kk in host[t]), t
    pools["graph"].step_many_device(d_acts, 0, K, use_graph=True)
    o = outputs(pools["graph"])
    assert all(o[kk].tobytes() == host[-1][kk].tobytes() for kk in host[-1])
    p = pools["rollout"]
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((K, n) + kk.shape, dtype=tdt[kk.dtype], device="cuda") for kk in p.keys]
    p.rollout_device(d_acts, K, cols)
    p.sync()
    for t in range(K):
        for kk, c in zip(p.keys, cols):
            assert c[t].cpu().numpy().tobytes() == host[t][kk.name].tobytes(), (t, kk.name)
    want = pools["step"].state_export().tobytes()
    for m in names[1:]:
        assert pools[m].state_export().tobytes() == want, m


def test_forced_budget_9(tmp_path):
    """ENVPOOL_B200_HC_PAIR_KS=9 (read once per process): the small-pool test in a subprocess,
    most rows of the crafted states in thread-local overflow."""
    env = dict(os.environ, **{FORCE: "9"})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "-p", "no:cacheprovider",
                        os.path.abspath(__file__) + "::test_small_pool_against_the_minimiser"],
                       env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "ks=9" in r.stdout, r.stdout[-3000:]
    print(r.stdout[-2500:])
