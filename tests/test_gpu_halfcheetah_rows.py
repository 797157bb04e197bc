"""GPU: HalfCheetah's two-lane kernel with constraint rows in its thread-local overflow.

hc_pair_kernel (csrc/mujoco.cu, csrc/mujoco_pair.cuh) keeps the first `ks` constraint rows of each
lane in dynamic shared memory, interleaved by thread, and rows ks..26 in a thread-local array.
ks follows the rows of a launch (epb_hc_pair_rows): 27 while one CTA per SM covers the batch, 10
at 32768 envs on a 132-SM H100, the benchmark's HalfCheetah configuration.  Resets and random
play rarely need more than a few rows per lane, so these tests press the cheetah into the floor
with its joints past their limits, and the CPU restatement of the pipeline (oracle/mjc_oracle.c)
shows that the crafted states need more rows than the budget under test.

Bars: integer and bool columns exact; float64 columns within 1e-9 relative-absolute per
teacher-forced env step (as test_gpu_halfcheetah.py); the float32 reward within 1e-6.  The entry
points that issue the same launch agree bit for bit; launches that differ only in the budget agree
to rounding (test_row_budget_sweep says why)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.gpu

MAXR, KS_MIN = 27, 9            # rows per lane at most; fewest ever held in shared memory
SWEEP = (9, 10, 14, 21, 27)     # forced budgets: the floor, the four the SM fit picks
EXACT = ("info:env_id", "info:players.env_id", "elapsed_step", "done", "discount", "step_type",
         "trunc")
FLOATS = ("obs", "info:reward_run", "info:reward_ctrl", "info:x_position", "info:x_velocity")
FORCE = "ENVPOOL_B200_HC_PAIR_KS"
# joint ranges of bthigh bshin bfoot fthigh fshin ffoot (half_cheetah.xml)
RANGE = np.array([[-.52, 1.05], [-.785, .785], [-.4, .785], [-1, .7], [-1.2, .87], [-.5, .5]])


def natural_rows(n, sms):
    """The budget the engine picks for a launch of n rows on `sms` SMs: 216 KB of shared memory
    per SM shared by the 64-thread CTAs one wave puts there (at most 4), a row being 10 doubles
    for each of the 64 threads."""
    ctas = -(-2 * n // 64)
    per_sm = min(max(-(-ctas // sms), 1), 4)
    return max(KS_MIN, min(MAXR, (216 * 1024 // per_sm) // (10 * 64 * 8)))


def lane_rows(J):
    """Lower bound on the rows each lane (back leg, front leg) of the kernel stores for the
    oracle's constraint Jacobian J [rows, 9].  Limit rows have a single +-1 entry.  The oracle
    writes 4 pyramid rows per contact, the kernel 3 (it merges the two +-y edges).  A row that
    touches dofs 3-5 is the back lane's, 6-8 the front lane's.  Root-only rows are contacts of the
    torso capsule (back lane) or the head capsule (front lane), two end spheres each: of k such
    contacts each capsule has at least k - 2."""
    nz = J != 0
    lim = nz.sum(1) == 1
    legs = (nz[:, 3:6].any(1), nz[:, 6:9].any(1))
    body0 = ~lim & ~legs[0] & ~legs[1]
    assert body0.sum() % 4 == 0 and all((~lim & leg).sum() % 4 == 0 for leg in legs)
    both = 3 * max(0, int(body0.sum()) // 4 - 2)
    return [int((lim & leg).sum()) + 3 * int((~lim & leg).sum()) // 4 + both for leg in legs]


def craft(count, seed, keep_above=10):
    """`count` states (qpos, qvel, qacc_warmstart) [count, 27] with a lane that needs more than
    `keep_above` rows, and their per-lane bounds [count, 2].  Every other candidate has the torso
    origin 0 .. 0.7 above the floor and leg joints in +-1.2 rad; the others lie flat, the torso
    0.1 .. 0.2 into the floor, every leg joint 0.05 .. 0.4 rad past one end of its range: up to
    all 27 rows a lane can have."""
    from oracle.oracle_lib import MjcSim, lib

    L = lib()
    L.mjc_warm_mut.restype = ctypes.POINTER(ctypes.c_double)
    L.mjc_warm_mut.argtypes = [ctypes.c_void_p]
    sim = MjcSim()
    warm = np.ctypeslib.as_array(L.mjc_warm_mut(sim.d), shape=(9,))
    rng = np.random.default_rng(seed)
    states, bounds = [], []
    while len(states) < count:
        q = np.zeros(9)
        q[0] = rng.uniform(-1, 1)
        if len(states) % 2:
            q[1] = rng.uniform(-0.7, 0.0)
            q[2] = rng.uniform(-0.3, 0.3)
            q[3:] = rng.uniform(-1.2, 1.2, 6)
        else:
            q[1] = rng.uniform(-0.9, -0.8)
            q[2] = rng.uniform(-0.1, 0.1)
            past = rng.uniform(0.05, 0.4, 6)
            q[3:] = np.where(rng.random(6) < 0.5, RANGE[:, 0] - past, RANGE[:, 1] + past)
        v, w = rng.normal(0, 0.5, 9), rng.normal(0, 2.0, 9)
        sim.qpos[:], sim.qvel[:], warm[:] = q, v, w
        b = lane_rows(sim.solve_problem()["J"])
        if max(b) > keep_above:
            states.append(np.concatenate([q, v, w]))
            bounds.append(b)
    return np.array(states), np.array(bounds)


def grid_rows(n):
    """Rows spread over a launch's grid (32 envs per CTA): the whole first CTA, every lane pair
    of its two warps; the last 33 rows, the last full CTA plus at n = 4097 the lone env of the
    partial one; every 37th row in between."""
    return np.unique(np.concatenate([np.arange(32), np.arange(n - 33, n),
                                     np.arange(32, n - 33, 37)]))


def place(pool, states, envs):
    """The pool's state blob with states[i % len(states)] in env envs[i]."""
    blob = pool.state_export()
    rs = pool.state_arrays(blob)["rstate"]
    rs[:27, envs] = states[np.arange(len(envs)) % len(states)].T
    return blob


def _relerr(g, w):
    g, w = g.astype(np.float64), w.astype(np.float64)
    return np.abs(g - w) / (1 + np.abs(w))


def forced_step(pool, orc, a, rows, env_ids=None, ctx=""):
    """One step of the pool on the batch (a, env_ids); the oracle, its envs first set to the
    pool's state, steps batch rows `rows` alone.  Returns (pool outputs, worst float64 error,
    the pool's state arrays before the step)."""
    ids = np.arange(len(a)) if env_ids is None else np.asarray(env_ids)
    st = pool.state_arrays(pool.state_export())
    rs, fl = st["rstate"], st["flags"]
    for e in ids[rows]:
        orc.mjc_set(e, rs[:27, e], int(fl[e] & 1), int(fl[e] >> 1))
    g = pool.step(a, env_ids)
    w = orc.step(a[rows], ids[rows])
    for k in EXACT:
        np.testing.assert_array_equal(g[k][rows], w[k], err_msg=f"{ctx} {k}")
    worst = 0.0
    for k in FLOATS:
        err = float(_relerr(g[k][rows], w[k]).max())
        assert err <= 1e-9, (ctx, k, err)
        worst = max(worst, err)
    assert _relerr(g["reward"][rows], w["reward"]).max() <= 1e-6, ctx
    return g, worst, st


def assert_bitwise(got, want, ctx, float_tol=0.0):
    """Every column equal bit for bit; with float_tol > 0, float64 columns within float_tol
    relative-absolute instead, and the float32 reward (rounded from such a float64) within 1e-6.
    Returns (worst float64 error, rows that are not bit-identical)."""
    assert set(got) == set(want), ctx
    worst, rows = 0.0, set()
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (ctx, k)
        if got[k].tobytes() == want[k].tobytes():
            continue
        bad = np.argwhere(np.asarray(got[k] != want[k]))
        if float_tol == 0.0 or want[k].dtype.kind != "f":
            raise AssertionError(f"{ctx}: {k} differs at {bad[:3].tolist()}")
        err = float(_relerr(got[k], want[k]).max())
        assert err <= (float_tol if want[k].dtype == np.float64 else 1e-6), (ctx, k, err)
        if want[k].dtype == np.float64:
            worst = max(worst, err)
        rows.update(bad[:, 0].tolist())
    return worst, rows


@pytest.fixture(scope="module")
def crafted():
    states, bounds = craft(240, seed=17)
    lanes = bounds.max(1)
    # the overflow array (18 rows at ks = 9) is used to its end, and every budget below 27 has
    # states that overflow it
    assert lanes.max() == MAXR, lanes.max()
    for ks in SWEEP[:-1]:
        assert (lanes > ks).sum() >= 8, (ks, np.bincount(lanes))
    return states, bounds


@pytest.fixture
def natural_budget():
    if FORCE in os.environ:
        pytest.skip(f"{FORCE} is set: these tests check the budget the engine picks itself")


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def budget_worker(out_dir):
    """One forced budget (ENVPOOL_B200_HC_PAIR_KS, read once per process): teacher-forced steps
    of a 4097-env pool with the crafted states spread over its grid; writes the outputs of every
    step and the final state to out_dir/ks<ks>.npz."""
    from envpool_b200 import _capi
    from oracle.oracle_lib import OraclePool

    ks = int(os.environ[FORCE])
    states = np.load(os.path.join(out_dir, "crafted.npz"))["states"]
    n, T = 4097, 6
    pool = _capi.CPool("HalfCheetah", n, seed=3, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=3, max_episode_steps=1000)
    assert [pool.hc_pair_rows(m) for m in (1, n)] == [ks, ks]
    pool.reset()
    orc.reset()
    rows = grid_rows(n)
    pool.state_import(place(pool, states, rows))
    checked = np.union1d(rows, np.arange(0, n, 16))
    rng = np.random.default_rng(5)
    out, worst = {}, 0.0
    for t in range(T):
        a = rng.uniform(-1.2, 1.2, size=(n, 6))
        g, err, _ = forced_step(pool, orc, a, checked, ctx=f"ks={ks} t={t}")
        worst = max(worst, err)
        out.update({f"{t}:{k}": v for k, v in g.items()})
    st = pool.state_arrays(pool.state_export())
    out.update({"state:rstate": st["rstate"].T, "state:flags": st["flags"],
                "state:mt_idx": st["mt_idx"]})
    np.savez(os.path.join(out_dir, f"ks{ks}.npz"), **out)
    with open(os.path.join(out_dir, f"ks{ks}.json"), "w") as fh:
        json.dump({"ks": ks, "worst": worst, "crafted_rows": len(rows)}, fh)


def test_row_budget_query(capi, natural_budget):
    sms = _sms()
    n = 32768
    hc = capi.CPool("HalfCheetah", n, seed=0, max_episode_steps=1000)
    sizes = (1, 4224, 4225, 6000, 8448, 8449, 12672, 12673, 32761, 32768)
    got = [hc.hc_pair_rows(m) for m in sizes]
    assert got == [natural_rows(m, sms) for m in sizes], (sms, got)
    if sms == 132:
        assert got == [27, 27, 21, 21, 21, 14, 14, 10, 10, 10], got
    assert hc.hc_pair_rows(0) == 0 and hc.hc_pair_rows(n + 1) == 0
    assert capi.CPool("CartPole", 64).hc_pair_rows() == 0


def test_row_budget_sweep(capi, crafted, tmp_path):
    """Every forced budget against the oracle and against each other.

    The budgets agree bit for bit in every integer and bool column and in all but a few envs,
    but not in all of them.  In the line search's later passes (mujoco_pair.cuh, the
    `for (int k = 1; k < cm.ls_iter; ++k)` loop) the overflow instantiation keeps the first
    three overflow rows in registers and hoists their D * jv * jv out of the search, so for those
    rows `d2o += D * jv * jv` is DMUL, DMUL, DADD in the sm_90a SASS; every other row, in the
    slab or in overflow, gets DMUL, DFMA.  Which rows are the first three in overflow depends on
    ks, so an env whose active rows include one of them takes a different last bit in d2o, and
    so in the Newton step of alpha.  That is rounding and nothing else: the float columns are
    held to 1e-12 relative-absolute against ks = 27 (measured: 3e-14 after 6 steps)."""
    states, bounds = crafted
    placed = bounds[np.arange(len(grid_rows(4097))) % len(states)].max(1)
    assert placed.max() == MAXR and all((placed > ks).any() for ks in SWEEP[:-1])
    np.savez(tmp_path / "crafted.npz", states=states)
    for ks in SWEEP:
        env = dict(os.environ, **{FORCE: str(ks)})
        r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           timeout=600)
        assert r.returncode == 0, (ks, r.stdout[-3000:])
    want = dict(np.load(tmp_path / f"ks{MAXR}.npz"))
    for ks in SWEEP:
        diff, envs = assert_bitwise(dict(np.load(tmp_path / f"ks{ks}.npz")), want,
                                    f"ks={ks} vs ks={MAXR}", float_tol=1e-12)
        with open(tmp_path / f"ks{ks}.json") as fh:
            info = json.load(fh)
        print(f"ks={ks}: lanes over budget {int((placed > ks).sum())}/{len(placed)}, "
              f"worst rel err vs oracle {info['worst']:.3e}, vs ks={MAXR} {diff:.1e} "
              f"({len(envs)} envs not bit-identical)")
    print("largest per-lane row bound placed:", int(placed.max()))


@pytest.mark.parametrize("n", [32768, 32761])
def test_benchmark_shape_through_every_entry_point(capi, crafted, natural_budget, n):
    """The benchmark's pool size at the budget the engine picks (10 on a 132-SM H100; 32761
    leaves the last CTA partial).  One state blob, K steps through each entry point: the same
    kernel at the same budget, so the same bits; the host path also against the oracle."""
    import torch
    from oracle.oracle_lib import OraclePool

    states, bounds = crafted
    sms = _sms()
    ks = natural_rows(n, sms)
    if sms == 132:
        assert ks == 10
    K = 12
    rng = np.random.default_rng(n)
    rows = np.union1d(np.r_[0:32, n - 33:n], rng.choice(n, 160, replace=False))
    placed = bounds[np.arange(len(rows)) % len(states)].max(1)
    assert placed.max() == MAXR and (placed > ks).sum() >= len(rows) // 2
    names = ("step", "step_device", "graph", "direct", "timed", "rollout")
    pools = {k: capi.CPool("HalfCheetah", n, seed=11, max_episode_steps=1000) for k in names}
    assert all(p.hc_pair_rows() == ks for p in pools.values())
    pools["step"].reset()
    blob = place(pools["step"], states, rows)
    for p in pools.values():
        p.state_import(blob)
    acts = rng.uniform(-1.2, 1.2, size=(K, n, 6))
    d_acts = torch.from_numpy(acts).cuda()

    orc = OraclePool("HalfCheetah", n, seed=11, max_episode_steps=1000)
    orc.reset()
    checked = np.union1d(rows, np.arange(0, n, 16))
    host, worst = [], 0.0
    for t in range(K):
        g, err, _ = forced_step(pools["step"], orc, acts[t], checked, ctx=f"n={n} t={t}")
        host.append(g)
        worst = max(worst, err)

    def outputs(p):
        p.sync()
        return {k: v.cpu().numpy() for k, v in p.outputs_torch().items()}

    dev = []
    for t in range(K):
        pools["step_device"].step_device(d_acts[t])
        dev.append(outputs(pools["step_device"]))
    pools["graph"].step_many_device(d_acts, 0, K, use_graph=True)
    pools["direct"].step_many_device(d_acts, 0, K, use_graph=False)
    assert pools["timed"].step_many_timed(d_acts, 0, K, 4, K) > 0   # as bench.py's Timer
    p = pools["rollout"]
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64, np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((K, n) + k.shape, dtype=tdt[k.dtype], device="cuda") for k in p.keys]
    p.rollout_device(d_acts, K, cols)
    p.sync()
    for t in range(K):
        assert_bitwise(dev[t], host[t], f"step_device t={t}")
        roll = {k.name: c[t].cpu().numpy() for k, c in zip(p.keys, cols)}
        assert_bitwise(roll, host[t], f"rollout_device t={t}")
    for name in ("graph", "direct", "timed"):
        assert_bitwise(outputs(pools[name]), host[-1], f"{name} t={K - 1}")
    want = pools["step"].state_export()
    for name in names[1:]:
        assert pools[name].state_export().tobytes() == want.tobytes(), name
    print(f"n={n}: ks={ks} on {sms} SMs, crafted rows {len(rows)} (largest per-lane bound "
          f"{int(placed.max())}, over budget {int((placed > ks).sum())}), "
          f"worst rel err vs oracle {worst:.3e}")


def test_batches_that_are_not_the_pool(capi, crafted, natural_budget):
    """A 32768-env pool stepped with a permuted full batch, then with a partial batch of 6000
    ids: the budget follows the batch rows (21 at 6000 on a 132-SM H100), envs outside the batch
    keep their state bit for bit."""
    from oracle.oracle_lib import OraclePool

    states, bounds = crafted
    sms = _sms()
    n = 32768
    pool = capi.CPool("HalfCheetah", n, seed=13, max_episode_steps=1000)
    orc = OraclePool("HalfCheetah", n, seed=13, max_episode_steps=1000)
    pool.reset()
    orc.reset()
    rng = np.random.default_rng(8)
    envs = rng.choice(n, 200, replace=False)
    pool.state_import(place(pool, states, envs))
    worst = 0.0

    perm = rng.permutation(n).astype(np.int32)
    assert pool.hc_pair_rows(n) == natural_rows(n, sms)
    rows = np.nonzero(np.isin(perm, np.union1d(envs, np.arange(0, n, 16))))[0]
    for t in range(3):
        a = rng.uniform(-1.2, 1.2, size=(n, 6))
        _, err, _ = forced_step(pool, orc, a, rows, perm, ctx=f"permuted t={t}")
        worst = max(worst, err)

    m = 6000
    ks = natural_rows(m, sms)
    if sms == 132:
        assert ks == 21
    assert pool.hc_pair_rows(m) == ks
    # half of the crafted envs, among them states that overflow this budget too
    assert (bounds[:100].max(1) > ks).any()
    rest = np.setdiff1d(np.arange(n), envs[:100])
    ids = np.concatenate([envs[:100], rng.choice(rest, m - 100, replace=False)]).astype(np.int32)
    rng.shuffle(ids)
    out = np.setdiff1d(np.arange(n), ids)
    for t in range(4):
        a = rng.uniform(-1.2, 1.2, size=(m, 6))
        _, err, before = forced_step(pool, orc, a, np.arange(m), ids, ctx=f"partial t={t}")
        worst = max(worst, err)
        after = pool.state_arrays(pool.state_export())
        for k, axis in (("rstate", 1), ("flags", 0), ("mt_idx", 0), ("mt", 1)):
            assert (np.take(after[k], out, axis).tobytes() ==
                    np.take(before[k], out, axis).tobytes()), (t, k)
    print(f"permuted full batch ks={pool.hc_pair_rows(n)}, partial batch of {m} ks={ks}; "
          f"worst rel err vs oracle {worst:.3e}")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    budget_worker(sys.argv[1])
