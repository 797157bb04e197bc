"""GPU: classic.cu's steps bit for bit against the host model of oracle/classic_model.py fed the
device's own sin / cos (classic_lib's probe of M<R>), in both precisions, and those sin / cos
values pinned on their own against a high-precision reference.

Every operation of a classic step other than sin / cos is an IEEE basic operation, and
classic.cu is built with -fmad=false, so a model doing the same operations in the same order
must match the kernels exactly: state bits, reward, flags and every output column.  The
crafted boundary cases of classic_cases.py (found with the device's sin / cos) go through every
entry point and every compiled step kernel; free-running runs cover a whole registered episode;
the benchmark's shapes are checked on a sample of envs."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import classic_cases as C
from helpers import REGISTERED, random_actions
from oracle import classic_model as M

pytestmark = pytest.mark.gpu
PRECISIONS = {"f64": np.float64, "f32": np.float32}
T_CRAFTED = 10   # the crafted step, then free-running steps with auto-resets


def _tdt():
    import torch

    return {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
            np.dtype(np.bool_): torch.bool}


def bits_equal(got, want, ctx):
    assert set(got) == set(want), (ctx, sorted(set(got) ^ set(want)))
    for k, w in want.items():
        g = np.ascontiguousarray(got[k])
        w = np.ascontiguousarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape, (ctx, k, g.dtype, w.dtype, g.shape,
                                                           w.shape)
        if g.tobytes() != w.tobytes():
            bad = np.flatnonzero((g.view(np.uint8) != w.view(np.uint8)).reshape(len(g), -1)
                                 .any(axis=1))
            raise AssertionError(f"{ctx} {k}: {bad.size} rows differ, first {bad[:5].tolist()}: "
                                 f"got {g[bad[:3]].tolist()} want {w[bad[:3]].tolist()}")


def outputs(pool, rows=None):
    return {k: (v if rows is None else v[rows]).cpu().numpy()
            for k, v in pool.outputs_torch().items()}


class Reference:
    """The device-provider model of a pool whose envs start from given states, stepping with the
    engine's auto-resets: the k-th reset of env e takes its record count[e] from Draws."""

    def __init__(self, task, R, state, cur, draws, count, env_ids=None):
        ms, _ = REGISTERED[task]
        self.model = M.ModelPool(task, R, M.DeviceTrig(), state, cur,
                                 np.zeros(len(cur), bool), ms, env_ids)
        self.draws, self.count = draws, count

    def _reset(self, rows):
        table = self.draws.upto(int(self.count[rows].max()) + 1)
        st = table[self.count[rows], rows]
        self.count[rows] += 1
        return st

    def run(self, acts):
        """outputs after every step, state and flags after the last"""
        return [self.model.step(a, self._reset) for a in acts]

    def flags(self):
        return ((self.model.cur << 1) | self.model.done).astype(np.int32)


def check_state(pool, ref, ctx, rows=slice(None)):
    st = pool.state_arrays(pool.state_export())
    got = np.ascontiguousarray(st["rstate"][:, rows].T)
    bits_equal({"rstate": got, "flags": st["flags"][rows]},
               {"rstate": ref.model.state, "flags": ref.flags()}, ctx)


def crafted_pool(capi, case, precision, seed=5):
    ms, iopt = REGISTERED[case.task]
    pool = capi.CPool(case.task, case.n, seed=seed, max_episode_steps=ms, iopt=iopt,
                      precision=precision)
    pool.reset_device()     # consumes record 0 of every env
    pool.sync()
    blob = pool.state_export()
    st = pool.state_arrays(blob)
    st["rstate"][:] = case.state.T
    st["flags"][:] = case.flags
    pool.state_import(blob)
    return pool


def crafted_run(task, precision, seed=5):
    """The crafted case (found with the device's sin / cos), its action stream and the
    reference outputs of every step."""
    R = PRECISIONS[precision]
    case = C.build(task, R, M.DeviceTrig())
    _, iopt = REGISTERED[task]
    acts = np.concatenate([case.act[None],
                           random_actions(task, np.random.default_rng(3), (T_CRAFTED - 1, case.n))
                           .reshape((T_CRAFTED - 1,) + case.act.shape)])
    draws = C.Draws(task, case.n, seed, iopt)
    ref = Reference(task, R, case.state, case.cur, draws, np.ones(case.n, np.int64))
    outs = ref.run(acts)
    return case, acts, outs, ref


def host_and_device_paths(capi, task, precision):
    """Host path and one step_device per step, every step's outputs and the final state."""
    import torch

    case, acts, outs, ref = crafted_run(task, precision)
    pool = crafted_pool(capi, case, precision)
    for t, a in enumerate(acts):
        bits_equal(pool.step(a), outs[t], f"{task} {precision} host t={t}")
    check_state(pool, ref, f"{task} {precision} host state")
    pool = crafted_pool(capi, case, precision)
    d_acts = torch.from_numpy(acts).cuda()
    for t in range(len(acts)):
        pool.step_device(d_acts[t])
        pool.sync()
        bits_equal(outputs(pool), outs[t], f"{task} {precision} step_device t={t}")
    check_state(pool, ref, f"{task} {precision} step_device state")
    return case, acts, outs, ref


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("task", C.CLASSIC)
def test_crafted_cases_through_every_entry_point(capi, task, precision):
    """Host path, step_device, the fused rollout, and captured, direct and timed step chains
    from the same crafted states: every output column of every step (the chains: of the last)
    and the exported state bits and flags against the device-provider model."""
    import torch

    case, acts, outs, ref = host_and_device_paths(capi, task, precision)
    d_acts = torch.from_numpy(acts).cuda()
    T, N = len(acts), case.n
    pool = crafted_pool(capi, case, precision)
    cols = [torch.empty((T, N) + k.shape, dtype=_tdt()[k.dtype], device="cuda")
            for k in pool.keys]
    pool.rollout_device(d_acts, T, cols)
    pool.sync()
    for t in range(T):
        got = {k.name: c[t].cpu().numpy() for k, c in zip(pool.keys, cols)}
        bits_equal(got, outs[t], f"{task} {precision} rollout t={t}")
    check_state(pool, ref, f"{task} {precision} rollout state")
    for how in ("graph", "direct", "timed"):
        p = crafted_pool(capi, case, precision)
        if how == "timed":
            assert p.step_many_timed(d_acts, 0, T, 2, T) > 0
        else:
            p.step_many_device(d_acts, 0, T, use_graph=how == "graph")
        p.sync()
        bits_equal(outputs(p), outs[-1], f"{task} {precision} {how} chain")
        check_state(p, ref, f"{task} {precision} {how} chain state")
        p.close()


_BLOCK = """
import sys
from envpool_b200 import _capi
import test_gpu_classic_model as G
_capi.load_library()
for task in G.C.CLASSIC:
    for precision in G.PRECISIONS:
        G.host_and_device_paths(_capi, task, precision)
print("BLOCK%s OK" % sys.argv[1])
"""


@pytest.mark.parametrize("block", [128])
def test_crafted_cases_on_the_wide_step_kernels_in_a_subprocess(capi, block):
    """ENVPOOL_B200_STEP_BLOCK is read once per process: a fresh interpreter steps every crafted
    case, both precisions, on the 128-thread step kernel (host path and step_device)."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, ENVPOOL_B200_STEP_BLOCK=str(block),
               PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]))
    r = subprocess.run([sys.executable, "-s", "-c", _BLOCK, str(block)], env=env, cwd=here,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and f"BLOCK{block} OK" in r.stdout, \
        r.stdout[-2000:] + r.stderr[-3000:]


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("task", C.CLASSIC)
def test_free_running_episode_bit_exact(capi, task, precision):
    """2048 envs for one full registered episode length (CartPole and Acrobot 500 steps,
    Pendulum and MountainCar 200, MountainCarContinuous 999) in one fused rollout: every row of
    every step and the final state bits against the device-provider model."""
    import torch

    n, seed = 2048, 9
    ms, iopt = REGISTERED[task]
    R = PRECISIONS[precision]
    draws = C.Draws(task, n, seed, iopt)
    ref = Reference(task, R, draws.upto(1)[0], np.zeros(n, np.int32), draws,
                    np.ones(n, np.int64))
    acts = random_actions(task, np.random.default_rng(4), (ms, n))
    pool = capi.CPool(task, n, seed=seed, max_episode_steps=ms, iopt=iopt, precision=precision)
    pool.reset_device()
    cols = [torch.empty((ms, n) + k.shape, dtype=_tdt()[k.dtype], device="cuda")
            for k in pool.keys]
    pool.rollout_device(torch.from_numpy(acts).cuda(), ms, cols)
    pool.sync()
    host = [c.cpu().numpy() for c in cols]
    for t in range(ms):
        want = ref.model.step(acts[t], ref._reset)
        got = {k.name: h[t] for k, h in zip(pool.keys, host)}
        bits_equal(got, want, f"{task} {precision} t={t}")
    check_state(pool, ref, f"{task} {precision} final state")


@pytest.mark.parametrize("task,n,steps", [("CartPole", 65536, 192), ("Pendulum", 1 << 20, 200),
                                          ("Acrobot", 1 << 20, 100)])
def test_benchmark_shapes_bit_exact(capi, task, n, steps):
    """bench.py's classic configurations in f64 (seed 0, registered limits): 16 steps of a direct
    chain, then one captured chain of `steps` steps.  The first and last 4096 envs and a strided
    sample, outputs and state bits, against the device-provider model seeded seed + env id."""
    import torch

    seed = 0
    ms, iopt = REGISTERED[task]
    rng = np.random.default_rng(8)
    acts = random_actions(task, rng, (64, n))
    d_acts = torch.from_numpy(acts).cuda()
    ids = np.unique(np.concatenate([np.arange(4096), np.arange(n - 4096, n),
                                    np.arange(4096, n - 4096, 1021)])).astype(np.int32)
    d_ids = torch.from_numpy(ids).long().cuda()
    draws = C.Draws(task, len(ids), seed, iopt, env_seed=ids + seed)
    ref = Reference(task, np.float64, draws.upto(1)[0], np.zeros(len(ids), np.int32), draws,
                    np.ones(len(ids), np.int64), env_ids=ids)
    pool = capi.CPool(task, n, seed=seed, max_episode_steps=ms, iopt=iopt)
    pool.reset_device()
    pool.step_many_device(d_acts, 0, 16, use_graph=False)
    pool.step_many_device(d_acts, 16, steps, use_graph=True)
    pool.sync()
    for t in range(16 + steps):
        want = ref.model.step(acts[t % 64][ids], ref._reset)
    bits_equal(outputs(pool, d_ids), want, f"{task} N={n}")
    check_state(pool, ref, f"{task} N={n} state", rows=ids)


# ---------------------------------------------------------------------------- trig accuracy
P_BITS = {"f64": (53, -1074), "f32": (24, -149)}
RANGES = {"CartPole theta": (-0.5, 0.5), "CartPole switch neighbourhood": (-3.0, 3.0),
          "Pendulum theta": (-math.pi, math.pi),
          "Acrobot theta1 - pi/2, theta1 + theta2 - pi/2, obs angles": (-8.0, 6.5),
          "MountainCar 3 pos": (-3.6, 1.8)}
DENSE, SUB = 1 << 20, 1 << 14


def crafted_args(R, lo, hi):
    """0, +-subnormals, +-the smallest normal, +-0.5 and its neighbours, and the values of R
    nearest k pi / 2 (with their neighbours) inside [lo, hi]."""
    fi = np.finfo(R)
    tiny_sub = np.array([fi.smallest_subnormal, fi.smallest_subnormal * 3,
                         fi.smallest_normal / 2, fi.smallest_normal], R)
    half = C.ulps(np.full(3, 0.5, R), np.array([-1, 0, 1]))
    xs = [np.zeros(1, R), tiny_sub, -tiny_sub, half, -half]
    for k in range(-6, 7):
        c = R(k * math.pi / 2)
        xs.append(C.ulps(np.full(3, c, R), np.array([-1, 0, 1])))
    x = np.concatenate(xs)
    return x[(x >= lo) & (x <= hi)]


def mp_ref(x):
    """sin and cos of every x at 60 digits, each as a double-double (hi, lo): [2 fns][2][n]."""
    import mpmath

    mpmath.mp.dps = 60
    out = np.empty((2, 2, len(x)))
    for i, v in enumerate(x.astype(np.float64)):
        m = mpmath.mpf(float(v))
        for j, f in enumerate((mpmath.sin, mpmath.cos)):
            r = f(m)
            out[j, 0, i] = float(r)
            out[j, 1, i] = float(r - out[j, 0, i])
    return out


def ulp_err(got, hi, lo, precision):
    """|got - (hi + lo)| in ulps of R at hi + lo (hi, lo: float64 or long double)."""
    p, emin = P_BITS[precision]
    m, e = np.frexp(hi)
    e = np.where((np.abs(m) == 0.5) & (np.sign(lo) == -np.sign(hi)), e - 1, e)
    ulp = np.ldexp(np.ones_like(hi), np.maximum(e.astype(np.int64), emin + p) - p)
    err = np.abs((got.astype(hi.dtype) - hi) - lo) / ulp
    exact_zero = (hi == 0) & (lo == 0)
    return np.where(exact_zero, np.where(got == 0, 0.0, np.inf), err).astype(np.float64)


def ld_ref(x, which):
    xl = x.astype(np.longdouble)
    return np.sin(xl) if which == "sin" else np.cos(xl)


@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_trig_accuracy_over_every_env_range(capi, precision):
    """classic.cu's M<R>::sincos_small_, sin_, cos_ and sincos_ over each env's argument range
    (2^20 dense points plus crafted arguments): the double sincos_small_ within 1 ulp on its
    polynomial's range |x| <= 0.5, everything else within 2 ulp (CUDA's sin, cos and sincos; on an
    H100 the double ones measured up to 1.42 ulp on these ranges), and sincos_ bitwise equal to
    (sin_, cos_).  The
    crafted arguments and a 2^14 subsample against mpmath at 60 digits; the dense points against
    numpy's long double, itself first held to mpmath within 1e-3 ulp on the subsample."""
    from oracle.classic_lib import device_trig

    assert np.finfo(np.longdouble).nmant >= 63, "needs x87 extended long double"
    R = PRECISIONS[precision]
    # The double sincos_small_'s own polynomial (|x| <= 0.5) is within 1 ulp; above 0.5 it is
    # CUDA's sincos.  The float one is sincosf throughout.
    def bound(rname, fn):
        return 1.0 if (precision, fn, rname) == ("f64", "sincos_small", "CartPole theta") else 2.0

    worst = {}
    for rname, (lo, hi) in RANGES.items():
        dense = np.linspace(lo, hi, DENSE).astype(R)
        craft = crafted_args(R, lo, hi)
        sub = dense[np.random.default_rng(0).choice(DENSE, SUB, replace=False)]
        ref_c, ref_s = mp_ref(craft), mp_ref(sub)
        vals = {}
        for fn in ("sincos_small", "sin", "cos", "sincos"):
            vals[fn] = [device_trig(fn, x) for x in (dense, craft, sub)]
        for part in range(3):
            s_, _ = vals["sin"][part]
            _, c_ = vals["cos"][part]
            ss, cc = vals["sincos"][part]
            assert ss.tobytes() == s_.tobytes() and cc.tobytes() == c_.tobytes(), \
                (precision, rname, "sincos_ differs from (sin_, cos_)")
        for fn in ("sincos_small", "sin", "cos", "sincos"):
            for which in ("sin", "cos"):
                if (fn, which) in (("sin", "cos"), ("cos", "sin")):
                    continue
                k = 0 if which == "sin" else 1
                got_d, got_c, got_s = (vals[fn][p][k] for p in range(3))
                e_mp_sub = ulp_err(got_s, ref_s[k, 0], ref_s[k, 1], precision)
                zero = np.zeros(len(sub), np.longdouble)
                e_ld_sub = ulp_err(got_s, ld_ref(sub, which), zero, precision)
                agree = np.abs(e_mp_sub - e_ld_sub).max()
                assert agree <= 1e-3, (precision, rname, fn, which, "long double vs mpmath",
                                       agree)
                e = max(ulp_err(got_c, ref_c[k, 0], ref_c[k, 1], precision).max(),
                        ulp_err(got_d, ld_ref(dense, which), np.zeros(DENSE, np.longdouble),
                                precision).max(), e_mp_sub.max())
                worst[(rname, fn, which)] = e
    print(f"\nmax ulp error of classic.cu's M<{'double' if precision == 'f64' else 'float'}>:")
    for (rname, fn, which), e in worst.items():
        print(f"  {fn + '_':14s} {which:3s}  {rname:58s} {e:.4f}")
    bad = {k: v for k, v in worst.items() if v > bound(k[0], k[1])}
    assert not bad, bad
