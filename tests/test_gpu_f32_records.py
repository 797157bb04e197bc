"""GPU: classic_control's f32 mode through the reset-ahead record rings, the step chains and the
fused rollout, with every initial state held bit-exact to the oracle in both precisions.

Every classic env draws its initial state in double and casts it to the state type R
(classic.cu: `(R)v[k]` in CartPole and Acrobot, `(R)__dadd_rn(...)` in Pendulum,
`(R)rng->uniform_real(...)` in MountainCar).  Env e's i-th initial state is therefore exactly the
oracle's i-th initial state in f64 mode and exactly np.float32 of it in f32 mode, so the rings
(common.cuh StateView::rec: record i in slot i % rec_q, uint8 counters rcons / rprod) are checked
bit for bit here, not through float32 observations.  Pendulum, MountainCar and
MountainCarContinuous keep two floats per f32 state: their 8-byte records go through the uint2
branch of load_rec_real / store_rec_real, which no f64 env uses.

With max_episode_steps <= 3 no env is ever more than three steps away from such an exactly known
state, and none of these envs can terminate within three steps of its reset range (Pendulum never
terminates).  So hundreds of f32 steps are held to the double oracle at the per-step f32 bar of
test_gpu_parity.py::test_teacher_forced_single_step (2e-5 relative-absolute), with every flag
exact.  Pendulum's raw angle is not compared: float pi (3.14159274) is above pi, so f32 wraps the
angle in a slightly different window.  Its outputs (cos, sin, theta_dot, reward) do not depend on
the window.  classic.cu is built with -fmad=false, so the same arithmetic through a different
entry point must give the same bits."""
import numpy as np
import pytest

from classic_cases import Draws
from helpers import EXACT_KEYS, REGISTERED, assert_batch_equal, random_actions

pytestmark = pytest.mark.gpu
CLASSIC = ["CartPole", "Pendulum", "Acrobot", "MountainCar", "MountainCarContinuous"]
NR = {"CartPole": 4, "Pendulum": 2, "Acrobot": 4, "MountainCar": 2, "MountainCarContinuous": 2}
ATOL = {"f32": 2e-5, "f64": 1e-6}   # relative-absolute, as in test_gpu_parity.py
CHAINS = (1, 2, 3, 7, 64, 7, 2, 64, 1)
T = 64                              # rows of the action stream, cycled


def _outputs(pool, n=None):
    return {k: v.cpu().numpy() for k, v in pool.outputs_torch(n).items()}


def _float_err(got, want):
    """Largest relative-absolute error over the float columns."""
    err = 0.0
    for k, w in want.items():
        if w.dtype.kind == "f" and k not in EXACT_KEYS:
            w64 = w.astype(np.float64)
            err = max(err, float((np.abs(got[k] - w64) / (1 + np.abs(w64))).max()))
    return err


def check_rings(st, draws, count, precision, ctx, rows=slice(None), full=False):
    """The rings of the envs `rows` of an exported state `st` against the draw oracle, where
    count[j] is the number of records env rows[j] has consumed (forced resets plus auto-resets):
    rcons == count % 256, 1 <= rprod - rcons <= rec_q (== rec_q when `full`), every valid slot
    rec[e, i % rec_q], i in [count, count + valid), holds record i bit for bit, and an env that
    has not stepped since its last reset holds record count - 1 in rstate."""
    real, bits = (np.float32, np.uint32) if precision == "f32" else (np.float64, np.uint64)
    rec = st["rec"][rows]
    q = rec.shape[1]
    rcons = st["rcons"][rows].astype(np.int64)
    rprod = st["rprod"][rows].astype(np.int64)
    bad = np.flatnonzero(rcons != count % 256)
    assert bad.size == 0, (ctx, "rcons", bad[:5].tolist(), rcons[bad[:5]].tolist(),
                           count[bad[:5]].tolist())
    valid = (rprod - rcons) & 255
    assert 1 <= valid.min() and valid.max() <= q, (ctx, "valid", int(valid.min()), int(valid.max()))
    if full:
        assert (valid == q).all(), (ctx, "ring not full", int(valid.min()))
    table = draws.upto(int((count + valid).max())).astype(real)
    envs = np.arange(count.shape[0])
    for j in range(q):
        e = envs[valid > j]
        i = count[e] + j
        got, want = rec[e, i % q], table[i, e]
        diff = np.flatnonzero((got.view(bits) != want.view(bits)).any(axis=1))
        assert diff.size == 0, (ctx, f"env {e[diff[0]]} record {i[diff[0]]} slot {i[diff[0]] % q}",
                                got[diff[0]].tolist(), want[diff[0]].tolist())
    fresh = envs[((st["flags"][rows] >> 1) == 0) & (count > 0)]
    got = np.ascontiguousarray(st["rstate"][:, rows][:, fresh].T)
    want = table[count[fresh] - 1, fresh]
    diff = np.flatnonzero((got.view(bits) != want.view(bits)).any(axis=1))
    assert diff.size == 0, (ctx, f"rstate of env {fresh[diff[0]]} after its reset",
                            got[diff[0]].tolist(), want[diff[0]].tolist())


def _state_equal(pool, a, b, ctx):
    """Two state blobs of `pool`'s layout bit-identical; names the first array that is not."""
    if np.array_equal(a, b):
        return
    sa, sb = pool.state_arrays(a), pool.state_arrays(b)
    for k in sa:
        if sa[k].tobytes() != sb[k].tobytes():
            where = np.argwhere(sa[k].view(np.uint8) != sb[k].view(np.uint8))[:3].tolist()
            raise AssertionError(f"{ctx}: state blobs differ in {k} at {where}")
    raise AssertionError(f"{ctx}: state blobs differ outside the named arrays")


class Canonical:
    """A state blob with every ring filled up: imported into a scratch pool (whose import
    refills) and exported again.  The draws are a function of the records consumed, so runs that
    refilled at different times compare equal, and a wrong record in a valid slot stays wrong."""

    def __init__(self, capi, task, n, precision):
        _, iopt = REGISTERED[task]
        self.pool = capi.CPool(task, n, seed=12345, iopt=iopt, precision=precision)

    def __call__(self, blob):
        self.pool.state_import(blob)
        return self.pool.state_export()


class DenseRun:
    """One engine pool beside the oracle, both stepped on the same cycled actions.  After every
    call the engine's outputs are compared with the oracle's (flags exact, float columns at the
    precision's bar) and its rings with the draw oracle.  out[t] keeps the outputs seen after
    step t, for bit-for-bit comparisons between entry points."""

    def __init__(self, capi, task, precision, ms, n, seed, draws=None):
        import torch
        from oracle.oracle_lib import OraclePool

        _, iopt = REGISTERED[task]
        self.task, self.precision, self.n = task, precision, n
        self.pool = capi.CPool(task, n, seed=seed, max_episode_steps=ms, iopt=iopt,
                               precision=precision)
        self.orc = OraclePool(task, n, seed=seed, max_episode_steps=ms, iopt=iopt)
        self.draws = draws or Draws(task, n, seed, iopt)
        self.acts = random_actions(task, np.random.default_rng(seed), (T, n))
        self.d_acts = torch.from_numpy(self.acts).cuda()
        self.count = np.zeros(n, np.int64)
        self.t = 0
        self.out = {}
        self.worst = 0.0

    def _seen(self, got, want, ctx):
        assert_batch_equal(got, want, self.task, ATOL[self.precision],
                           f"{self.task} {self.precision} {ctx}")
        self.worst = max(self.worst, _float_err(got, want))
        self.out[self.t] = got

    def _oracle_step(self):
        want = self.orc.step(self.acts[self.t % T])
        self.count += want["elapsed_step"] == 0
        self.t += 1
        return want

    def rings(self, ctx, full=False):
        st = self.pool.state_arrays(self.pool.state_export())
        check_rings(st, self.draws, self.count, self.precision,
                    f"{self.task} {self.precision} {ctx}", full=full)

    def reset(self, host=False):
        if host:
            got = self.pool.reset()
        else:
            self.pool.reset_device()
            self.pool.sync()
            got = _outputs(self.pool)
        want = self.orc.reset()
        self.count += 1
        self._seen(got, want, "reset")
        self.rings("after the reset")

    def chain(self, K, graph=True, timed=False):
        if timed:
            self.pool.step_many_timed(self.d_acts, self.t % T, K, K // 2, K, use_graph=graph)
        else:
            self.pool.step_many_device(self.d_acts, self.t % T, K, use_graph=graph)
        for _ in range(K):
            want = self._oracle_step()
        self.pool.sync()
        ctx = f"{'graph' if graph else 'direct'}{' timed' if timed else ''} chain K={K} to t={self.t}"
        self._seen(_outputs(self.pool), want, ctx)
        self.rings(ctx, full=graph)   # a captured chain ends with a refill

    def steps(self, k, host=False):
        for _ in range(k):
            if host:
                got = self.pool.step(self.acts[self.t % T])
            else:
                self.pool.step_device(self.d_acts[self.t % T])
            want = self._oracle_step()
            if host:
                self._seen(got, want, f"host step to t={self.t}")
        if not host:
            self.pool.sync()
            self._seen(_outputs(self.pool), want, f"device steps to t={self.t}")
        self.rings(f"{k} {'host' if host else 'device'} steps to t={self.t}")

    def rollout(self, k):
        import torch

        tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
               np.dtype(np.bool_): torch.bool}
        # built on the host: a torch gather on the device would race the pool's own stream
        d = torch.from_numpy(np.ascontiguousarray(
            self.acts[(self.t + np.arange(k)) % T])).cuda()
        cols = [torch.empty((k, self.n) + key.shape, dtype=tdt[key.dtype], device="cuda")
                for key in self.pool.keys]
        self.pool.rollout_device(d, k, cols)
        self.pool.sync()
        host = [c.cpu().numpy() for c in cols]
        for r in range(k):
            want = self._oracle_step()
            self._seen({key.name: h[r] for key, h in zip(self.pool.keys, host)}, want,
                       f"rollout row {r} of {k} (t={self.t})")
        self.rings(f"rollout of {k} to t={self.t}", full=True)   # it leaves the rings full


@pytest.mark.parametrize("precision", ["f64", "f32"])
@pytest.mark.parametrize("task", CLASSIC)
def test_rings_hold_the_oracle_initial_states_bit_exact(capi, task, precision):
    """Right after pool creation, after the first forced reset, after captured chains with
    dense resets, and after forced resets and steps of partial id sets (host and device path),
    every valid ring slot is the oracle's initial state of that index, bit for bit, and rcons
    counts every record consumed."""
    import torch

    N = 2500
    run = DenseRun(capi, task, precision, 2, N, seed=11)
    run.rings("at creation", full=True)
    run.reset()
    for K in CHAINS:
        run.chain(K)
    rng = np.random.default_rng(4)
    for r in range(4):
        sub = np.sort(rng.choice(N, size=700, replace=False)).astype(np.int32)
        if r % 2:
            run.pool.reset_device(torch.from_numpy(sub).cuda())
            run.pool.sync()
            got = _outputs(run.pool, len(sub))
        else:
            got = run.pool.reset(sub)
        want = run.orc.reset(sub)
        run.count[sub] += 1
        assert_batch_equal(got, want, task, ATOL[precision], f"partial forced reset {r}")
        run.rings(f"partial forced reset {r}")
        sub = np.sort(rng.choice(N, size=900, replace=False)).astype(np.int32)
        a = random_actions(task, rng, (len(sub),))
        got, want = run.pool.step(a, sub), run.orc.step(a, sub)
        run.count[sub] += want["elapsed_step"] == 0
        assert_batch_equal(got, want, task, ATOL[precision], f"partial step {r}")
        run.rings(f"partial step {r}")


@pytest.mark.parametrize("ms", [1, 2, 3])
@pytest.mark.parametrize("task", CLASSIC)
def test_f32_dense_reset_chains_match_oracle_through_every_entry_point(capi, task, ms):
    """f32 step chains K = 1, 2, 3, 7, 64, 7, 2, 64, 1 replayed from CUDA graphs (the refill on
    its parallel branch) against the double oracle on a 2500-env pool (no multiple of a CTA).
    Then the same actions through direct chains, one step_device per step, host step(), the
    fused rollout in pieces of 64, 37 and 50 steps, and timed chains: each must reproduce the
    graph chain's outputs and (rings filled up) its state blob bit for bit."""
    N, seed = 2500, 11
    ref = DenseRun(capi, task, "f32", ms, N, seed)
    ref.reset()
    for K in CHAINS:
        ref.chain(K)
    print(f"{task} f32 ms={ms}: largest float error against the oracle {ref.worst:.2e}")
    canon = Canonical(capi, task, N, "f32")
    want_blob = canon(ref.pool.state_export())

    def direct(r):
        r.reset()
        for K in CHAINS:
            r.chain(K, graph=False)

    def device_steps(r):
        r.reset()
        for K in CHAINS:
            r.steps(K)

    def host_steps(r):
        r.reset(host=True)
        for K in CHAINS:
            r.steps(K, host=True)

    def rollout(r):
        r.reset()
        for k in (64, 37, 50):
            r.rollout(k)

    def timed(r):
        r.reset()
        for K in CHAINS:
            r.chain(K, timed=True)

    for drive in (direct, device_steps, host_steps, rollout, timed):
        run = DenseRun(capi, task, "f32", ms, N, seed, draws=ref.draws)
        drive(run)
        assert run.t == ref.t
        for t in sorted(set(ref.out) & set(run.out)):
            assert_batch_equal(run.out[t], ref.out[t], task, 0.0, f"{drive.__name__} t={t}")
        assert set(ref.out) <= set(run.out), (drive.__name__, sorted(set(ref.out) - set(run.out)))
        _state_equal(canon.pool, canon(run.pool.state_export()), want_blob, drive.__name__)


@pytest.mark.parametrize("ring", [None, (4, 2), (8, 6), (16, 14)])
@pytest.mark.parametrize("task", ["Pendulum", "Acrobot"])
def test_f32_ring_bound_under_the_tightest_reset_spacing(capi, monkeypatch, task, ring):
    """max_episode_steps = 1 in f32, 8-byte (Pendulum) and 16-byte (Acrobot) records: the
    default ring (16 records, refill every 8 steps), the smallest (4 / 2), 8 / 6 and the longest
    period a 16-ring allows (14), in captured chains and then 9 direct launches (the refill on
    the step's own stream), against the oracle and the draw oracle."""
    if ring:
        monkeypatch.setenv("ENVPOOL_B200_REC_Q", str(ring[0]))
        monkeypatch.setenv("ENVPOOL_B200_REFILL_EVERY", str(ring[1]))
    run = DenseRun(capi, task, "f32", 1, 5000, seed=2)
    if ring:
        assert run.pool.state_layout()["rec_q"] == ring[0]
    run.reset()
    for K in (64, 37, 64, 5, 64):
        run.chain(K)
    for _ in range(9):
        run.steps(1)
    print(f"{task} f32 ring={ring}: largest float error against the oracle {run.worst:.2e}")


@pytest.mark.parametrize("task", ["MountainCar", "Pendulum"])
def test_f32_counters_wrap_through_rollouts_and_single_steps(capi, task):
    """max_episode_steps = 1 for 684 steps: about 340 records per env, so the uint8 counters
    rcons / rprod pass 255.  Fused rollouts (which take the ring's records first, then draw in
    place, then redraw the ring) alternate with device and host single steps.  A state drawn in
    place is a record produced and consumed: the counters must still count every reset."""
    run = DenseRun(capi, task, "f32", 1, 1000, seed=5)
    run.reset()
    plan = [("roll", 64), ("dev", 5), ("roll", 37), ("host", 4), ("roll", 128), ("dev", 9),
            ("roll", 1), ("host", 3), ("roll", 96), ("dev", 2), ("roll", 200), ("host", 1),
            ("roll", 77), ("dev", 7), ("roll", 50)]
    for what, k in plan:
        if what == "roll":
            run.rollout(k)
        else:
            run.steps(k, host=what == "host")
    assert run.t == 684 and run.count.min() > 300, (run.t, int(run.count.min()))
    print(f"{task} f32 wrap: largest float error against the oracle {run.worst:.2e}")


@pytest.mark.parametrize("task", CLASSIC)
def test_f32_snapshot_mid_ring(capi, task):
    """An f32 state blob exported while the rings are partly consumed, imported into a fresh f32
    pool built with another seed, continues bit for bit.  A blob of the other precision is
    refused and leaves the pool's state as it was."""
    N, ms, seed = 1000, 3, 4
    _, iopt = REGISTERED[task]
    a = DenseRun(capi, task, "f32", ms, N, seed)
    b = DenseRun(capi, task, "f32", ms, N, seed)   # same history, then its pool is replaced
    for r in (a, b):
        r.reset(host=True)
        r.steps(13, host=True)
    st = a.pool.state_arrays(a.pool.state_export())
    q = st["rec"].shape[1]
    assert (((st["rprod"].astype(int) - st["rcons"]) & 255) < q).any(), "rings not consumed"
    blob = a.pool.state_export()
    b.pool = capi.CPool(task, N, seed=999, max_episode_steps=ms, iopt=iopt, precision="f32")
    f64 = capi.CPool(task, N, seed=seed, max_episode_steps=ms, iopt=iopt, precision="f64")
    before = b.pool.state_export()
    with pytest.raises(ValueError):
        b.pool.state_import(f64.state_export())
    assert np.array_equal(b.pool.state_export(), before)
    before = f64.state_export()
    with pytest.raises(ValueError):
        f64.state_import(blob)
    assert np.array_equal(f64.state_export(), before)
    b.pool.state_import(blob)
    b.rings("after the import", full=True)
    for r in (a, b):
        r.steps(20, host=True)
        r.chain(7)
        r.steps(5)
        r.rollout(30)
        r.chain(64, graph=False)
    for t in sorted(a.out):
        assert_batch_equal(b.out[t], a.out[t], task, 0.0, f"after the import t={t}")
    canon = Canonical(capi, task, N, "f32")
    _state_equal(canon.pool, canon(b.pool.state_export()), canon(a.pool.state_export()),
                 "imported pool")


@pytest.mark.parametrize("task", ["CartPole", "Pendulum"])
def test_f32_wide_cta_prefix_suffix_and_halves(capi, task):
    """N = 300000 > 132 SMs * 8 * 128: the 128-thread step kernel.  24 f32 steps in captured
    chains; the first and the last 4096 envs against the oracle (the last with env_seed =
    seed + env id), their rings against the draw oracle, and two env_id_offset halves (150000
    envs each, also on the 128-thread kernel) reproduce the full pool's outputs and state bit
    for bit."""
    import torch
    from oracle.oracle_lib import OraclePool

    _, iopt = REGISTERED[task]
    N, P, ms, seed = 300000, 4096, 3, 1
    H = N // 2

    def make(n, **kw):
        return capi.CPool(task, n, seed=seed, max_episode_steps=ms, iopt=iopt, precision="f32",
                          **kw)

    full, lo, hi = make(N), make(H), make(H, env_id_offset=H)
    suf_seed = seed + np.arange(N - P, N, dtype=np.int32)
    orcs = {"prefix": OraclePool(task, P, seed=seed, max_episode_steps=ms, iopt=iopt),
            "suffix": OraclePool(task, P, max_episode_steps=ms, iopt=iopt, env_seed=suf_seed)}
    draws = {"prefix": Draws(task, P, seed, iopt),
             "suffix": Draws(task, P, seed, iopt, env_seed=suf_seed)}
    rows = {"prefix": slice(0, P), "suffix": slice(N - P, N)}
    count = {k: np.ones(P, np.int64) for k in rows}
    acts = random_actions(task, np.random.default_rng(6), (24, N))
    d_acts = {full: torch.from_numpy(acts).cuda(),
              lo: torch.from_numpy(np.ascontiguousarray(acts[:, :H])).cuda(),
              hi: torch.from_numpy(np.ascontiguousarray(acts[:, H:])).cuda()}
    for p in d_acts:
        p.reset_device()
    want = {k: o.reset() for k, o in orcs.items()}
    t, worst = 0, 0.0
    for K in (5, 3, 16):
        for p, d in d_acts.items():
            p.step_many_device(d, t, K, use_graph=True)
        for k in range(K):
            for name, o in orcs.items():
                want[name] = o.step(acts[t + k][rows[name]])
                count[name] += want[name]["elapsed_step"] == 0
        t += K
        for p in d_acts:
            p.sync()
        f, l, h = _outputs(full), _outputs(lo), _outputs(hi)
        for k in f:
            assert np.array_equal(f[k][:H], l[k]), (task, t, k, "lo half")
            assert np.array_equal(f[k][H:], h[k]), (task, t, k, "hi half")
        for name in orcs:
            w = dict(want[name])
            for k in ("info:env_id", "info:players.env_id"):
                w[k] = w[k] + rows[name].start
            got = {k: v[rows[name]] for k, v in f.items()}
            assert_batch_equal(got, w, task, ATOL["f32"], f"{task} {name} t={t}")
            worst = max(worst, _float_err(got, w))
    print(f"{task} f32 N={N}: largest float error against the oracle {worst:.2e}")
    sf = full.state_arrays(full.state_export())
    for name in rows:
        check_rings(sf, draws[name], count[name], "f32", f"{task} {name}", rows=rows[name],
                    full=True)
    for half, sl in ((lo, slice(0, H)), (hi, slice(H, N))):
        sh = half.state_arrays(half.state_export())
        for k, v in sh.items():
            whole = sf[k][:, sl] if k in ("mt", "istate", "rstate") else sf[k][sl]
            assert np.array_equal(np.ascontiguousarray(whole).view(np.uint8), v.view(np.uint8)), \
                (task, k, sl)


def test_benchmark_timed_chain_matches_step_chain_f64(capi):
    """The chain bench.py times (CartPole, 65536 envs, f64, 128 untimed + 64 timed steps behind
    direct warm-up launches), captured and direct, leaves the outputs and the state blob
    bit-identical to the same steps through step_many_device, and a prefix matches the oracle."""
    import torch
    from oracle.oracle_lib import OraclePool

    task, N, P, lead, K = "CartPole", 65536, 4096, 128, 64
    ms, iopt = REGISTERED[task]
    acts = random_actions(task, np.random.default_rng(10), (T, N))
    d_acts = torch.from_numpy(acts).cuda()
    timed, plain = (capi.CPool(task, N, seed=0, max_episode_steps=ms, iopt=iopt)
                    for _ in range(2))
    orc = OraclePool(task, P, seed=0, max_episode_steps=ms, iopt=iopt)
    orc.reset()
    for p in (timed, plain):
        p.reset_device()
        p.step_many_device(d_acts, 0, 16, use_graph=False)
    t = 16
    for k in range(t):
        orc.step(acts[k % T][:P])
    for graph in (True, False):
        ms_timed = timed.step_many_timed(d_acts, t % T, lead + K, lead, lead + K,
                                         use_graph=graph)
        assert ms_timed > 0, ms_timed
        plain.step_many_device(d_acts, t % T, lead + K, use_graph=graph)
        for k in range(t, t + lead + K):
            want = orc.step(acts[k % T][:P])
        t += lead + K
        timed.sync()
        plain.sync()
        got = _outputs(timed)
        assert_batch_equal(got, _outputs(plain), task, 0.0, f"graph={graph}")
        assert_batch_equal({k: v[:P] for k, v in got.items()}, want, task, ATOL["f64"],
                           f"graph={graph} prefix")
        _state_equal(plain, timed.state_export(), plain.state_export(), f"graph={graph}")
