"""GPU: PGX TicTacToe-v1 and ConnectFour-v1, the engine's two-player kinds, bit for bit against
the C restatement (oracle/pgx_oracle.c), the reference's own thread pool (oracle/_ref, when
build() made it) and the fixtures recorded from it (tests/golden/pgx/), through every entry
point: the host path (sync, async, permuted and partial batches), the pybind `_send` with
explicit players.env_id rows, make_gymnasium / make_dm, step_device, the step chains (graph and
direct), the timed chain, the fused rollout, snapshots, the 64- and 128-thread step kernels and
the peer exchange."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import GOLDEN

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import pgx_lib  # noqa: E402
from oracle.pgx_lib import ACTIONS, PgxOracle, PgxRef, first_player_actions  # noqa: E402

pytestmark = pytest.mark.gpu
GAMES = ["TicTacToe", "ConnectFour"]
TASK_ID = {"TicTacToe": "TicTacToe-v1", "ConnectFour": "ConnectFour-v1"}
I32 = np.iinfo(np.int32)
FIXTURES = sorted(glob.glob(os.path.join(GOLDEN, "pgx", "*.npz")))


def flat(out):
    """A CPool batch ([n, 2, ...] per-player columns) as the reference's rows ([2 n, ...])."""
    return {k: (v.reshape((-1,) + v.shape[2:]) if k in PER_PLAYER else v)
            for k, v in out.items()}


PER_PLAYER = ("info:players.env_id", "reward", "discount", "obs", "info:players.id")


def assert_same(got, want, ctx):
    got = flat(got)
    for k, w in want.items():
        g = np.asarray(got[k])
        assert g.shape == w.shape and g.dtype == w.dtype, (ctx, k, g.shape, w.shape, g.dtype)
        if not np.array_equal(g, w):
            bad = np.argwhere(np.asarray(g != w).reshape(len(w), -1).any(1)).ravel()[:5]
            raise AssertionError(f"{ctx}: `{k}` differs in rows {bad.tolist()}")


def policy(game, rng, mask, legal_share=0.5):
    """Per env: a random legal action with probability legal_share, else one over the whole int32
    range (in range, -1, the action count, INT_MIN, INT_MAX)."""
    n, A = mask.shape
    a = rng.integers(-1, A + 1, size=n)
    special = rng.random(n) < 0.05
    a = np.where(special, np.array([I32.min, I32.max])[rng.integers(0, 2, size=n)], a)
    legal = np.array([rng.choice(np.flatnonzero(m)) for m in mask]) if legal_share > 0 else a
    return np.where(rng.random(n) < legal_share, legal, a).astype(np.int32)


def legal_fast(rng, mask):
    """A uniformly random legal action per env (vectorised: argmax of masked noise)."""
    return np.argmax(np.where(mask, rng.random(mask.shape), -1.0), axis=1).astype(np.int32)


@pytest.mark.parametrize("game", GAMES)
def test_random_and_legal_play_against_oracle_and_ref(capi, game):
    n, T = 2048, 1000
    pool = capi.CPool(game, n, seed=7)
    orc = PgxOracle(game, n, seed=7)
    ref = PgxRef(game, n, seed=7) if pgx_lib.ref_available() else None
    want = orc.reset()
    assert_same(pool.reset(), want, f"{game} reset")
    if ref is not None:
        assert_same(flat_ref(ref.reset()), want, f"{game} ref reset")
    rng = np.random.default_rng(1)
    for t in range(T):
        mask = want["info:legal_action_mask"]
        a = legal_fast(rng, mask) if t % 2 else policy(game, rng, mask, legal_share=0.0)
        want = orc.step(a)
        assert_same(pool.step(a), want, f"{game} step {t}")
        if ref is not None:
            assert_same(flat_ref(ref.step(a)), want, f"{game} ref step {t}")


def flat_ref(out):
    """Reference rows are already [2 n, ...]: give them CPool's [n, 2, ...] shape for flat()."""
    return {k: (v.reshape((-1, 2) + v.shape[1:]) if k in PER_PLAYER else v) for k, v in out.items()}


def load_fixture(path):
    z = np.load(path)
    meta = json.loads(str(z["meta"]))
    return meta, {k: z[k] for k in z.files if k != "meta"}


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_host_path(capi, path):
    meta, data = load_fixture(path)
    pool = capi.CPool(meta["game"], meta["num_envs"], seed=meta["seed"])
    keys = [k for k in data if k != "action"]
    assert_same(pool.reset(), {k: data[k][0] for k in keys}, "reset")
    for t, a in enumerate(data["action"]):
        assert_same(pool.step(a), {k: data[k][t + 1] for k in keys}, f"step {t}")


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_gymnasium_and_dm(path):
    import envpool_b200

    meta, data = load_fixture(path)
    task = TASK_ID[meta["game"]]
    n = meta["num_envs"]
    gym = envpool_b200.make_gymnasium(task, num_envs=n, seed=meta["seed"])
    dm = envpool_b200.make_dm(task, num_envs=n, seed=meta["seed"])
    obs, info = gym.reset()
    ts = dm.reset()
    assert np.array_equal(obs, data["obs"][0]) and np.array_equal(ts.observation.obs, data["obs"][0])
    assert np.array_equal(info["players"]["env_id"], data["info:players.env_id"][0])
    for t, a in enumerate(data["action"]):
        obs, rew, term, trunc, info = gym.step(a)
        ts = dm.step(a)
        w = {k: data[k][t + 1] for k in data if k != "action"}
        assert np.array_equal(obs, w["obs"]) and np.array_equal(rew, w["reward"]), t
        assert np.array_equal(term | trunc, w["done"]) and not trunc.any(), t
        assert np.array_equal(info["board"], w["info:board"]), t
        assert np.array_equal(info["current_player"], w["info:current_player"]), t
        assert np.array_equal(info["legal_action_mask"], w["info:legal_action_mask"]), t
        assert np.array_equal(info["players"]["id"], w["info:players.id"]), t
        assert np.array_equal(ts.observation.obs, w["obs"]), t
        assert np.array_equal(ts.reward, w["reward"]) and np.array_equal(ts.discount, w["discount"])
        assert np.array_equal(ts.step_type, w["step_type"]), t


@pytest.mark.parametrize("game", GAMES)
def test_max_num_players_must_be_two(game):
    import envpool_b200

    with pytest.raises(ValueError, match="max_num_players"):
        envpool_b200.make_gymnasium(TASK_ID[game], num_envs=4, max_num_players=1)


def torch_out(pool, n=None):
    return {k: v.cpu().numpy() for k, v in pool.outputs_torch(n).items()}


@pytest.mark.parametrize("game", GAMES)
def test_every_entry_point_gives_the_same_outputs_and_state(capi, game):
    import torch

    n, T, K = 3000, 16, 40
    rng = np.random.default_rng(5)
    orc = PgxOracle(game, n, seed=11)
    want = [orc.reset()]
    acts = np.empty((T, n), np.int32)
    for k in range(K):  # the stream: legal-random actions of the oracle's own trajectory
        if k < T:
            acts[k] = np.where(rng.random(n) < 0.9, legal_fast(rng, want[-1]["info:legal_action_mask"]),
                               rng.integers(-1, ACTIONS[game] + 1, size=n)).astype(np.int32)
        want.append(orc.step(acts[k % T]))
    d_acts = torch.from_numpy(acts).cuda()

    def fresh():
        p = capi.CPool(game, n, seed=11)
        p.reset_device()
        return p

    blobs = {}
    p = capi.CPool(game, n, seed=11)  # host path
    assert_same(p.reset(), want[0], "host reset")
    for k in range(K):
        assert_same(p.step(acts[k % T]), want[k + 1], f"host step {k}")
    blobs["host"] = p.state_export()
    p = fresh()  # step_device, one launch per step
    for k in range(K):
        p.step_device(d_acts[k % T])
        assert_same(torch_out(p), want[k + 1], f"step_device {k}")
    blobs["step_device"] = p.state_export()
    for name, graph in (("graph", True), ("direct", False)):
        p = fresh()
        p.step_many_device(d_acts, 0, K, use_graph=graph)
        torch.cuda.synchronize()
        assert_same(torch_out(p), want[K], f"step_many_device {name}")
        blobs[name] = p.state_export()
    p = fresh()
    assert p.step_many_timed(d_acts, 0, K, 4, K) > 0
    assert_same(torch_out(p), want[K], "step_many_timed")
    blobs["timed"] = p.state_export()
    p = fresh()
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((T, n) + k.shape, dtype=tdt[k.dtype], device="cuda") for k in p.keys]
    for r in range((K + T - 1) // T):  # rollouts of T steps, the last one shorter
        steps = min(T, K - r * T)
        p.rollout_device(d_acts[:steps].contiguous(), steps, cols)
        torch.cuda.synchronize()
        for t in range(steps):
            assert_same({k.name: c[t].cpu().numpy() for k, c in zip(p.keys, cols)},
                        want[r * T + t + 1], f"rollout step {r * T + t}")
    blobs["rollout"] = p.state_export()
    for name, b in blobs.items():
        assert np.array_equal(b, blobs["host"]), name


@pytest.mark.parametrize("game", GAMES)
def test_async_permuted_and_partial_batches(capi, game):
    n, B = 1000, 250
    rng = np.random.default_rng(9)
    pool = capi.CPool(game, n, seed=3, batch_size=B)
    orc = PgxOracle(game, n, seed=3)
    pool.reset_async()
    want = orc.reset()
    for b in range(n // B):
        assert_same(pool.recv(), {k: v[b * B * (2 if k in PER_PLAYER else 1):
                                        (b + 1) * B * (2 if k in PER_PLAYER else 1)]
                                  for k, v in want.items()}, f"async reset batch {b}")
    mask = want["info:legal_action_mask"].copy()
    for t in range(60):
        ids = rng.permutation(n).astype(np.int32)[:B]
        a = policy(game, rng, mask[ids], legal_share=0.7)
        pool.send(a, ids)
        w = orc.step(a, ids)
        assert_same(pool.recv(), w, f"async permuted step {t}")
        mask[ids] = w["info:legal_action_mask"]
    sync = capi.CPool(game, n, seed=4)
    orc = PgxOracle(game, n, seed=4)
    assert_same(sync.reset(), orc.reset(), "sync reset")
    mask = np.ones((n, ACTIONS[game]), bool)
    for t in range(60):
        m = int(rng.integers(1, n + 1))
        ids = rng.permutation(n).astype(np.int32)[:m]
        a = policy(game, rng, mask[ids])
        w = orc.step(a, ids)
        assert_same(sync.step(a, ids), w, f"partial batch of {m}, step {t}")
        mask[ids] = w["info:legal_action_mask"]


@pytest.mark.parametrize("game", GAMES)
def test_explicit_players_env_id(game):
    """`_send([env_id, players.env_id, action])`: each env acts with its first player row, in
    any order and with duplicates; an env without a player row raises."""
    import envpool_b200

    n = 64
    rng = np.random.default_rng(2)
    env = envpool_b200.make_gymnasium(TASK_ID[game], num_envs=n, seed=5)
    orc = PgxOracle(game, n, seed=5)
    ref = PgxRef(game, n, seed=5) if pgx_lib.ref_available() else None
    env.reset()
    want = orc.reset()
    if ref is not None:
        ref.reset()
    ids = np.arange(n, dtype=np.int32)
    for t in range(80):
        pids = np.concatenate([ids, ids[rng.integers(0, n, size=n // 2)]])  # duplicates
        pids = pids[rng.permutation(len(pids))].astype(np.int32)
        acts = policy(game, rng, want["info:legal_action_mask"][pids], legal_share=0.8)
        a = first_player_actions(ids, pids, acts)
        want = orc.step(a)
        env._send([ids, pids, acts])
        got = env._recv()
        for k, g in zip(env._state_keys, got):
            assert np.array_equal(g, want[k]), (t, k)
        if ref is not None:
            r = ref.step(acts, ids, pids)
            for k in want:
                assert np.array_equal(r[k], want[k]), ("ref", t, k)
    # the dict form and the inferred mapping (one action per env; two per env repeat env_id)
    obs, *_ = env.step({"action": np.zeros(2 * n, np.int32)})
    assert obs.shape[0] == 2 * n
    pids = np.arange(n - 1, dtype=np.int32)  # env n - 1 has no player row
    with pytest.raises(ValueError, match="no row in players.env_id"):
        env._send([ids, pids, np.zeros(n - 1, np.int32)])


@pytest.mark.parametrize("game", GAMES)
def test_snapshot_continues_in_a_pool_with_another_seed(capi, game):
    n = 777
    rng = np.random.default_rng(4)
    a_pool = capi.CPool(game, n, seed=21)
    orc = PgxOracle(game, n, seed=21)
    want = orc.reset()
    a_pool.reset()
    for _ in range(9):
        a = legal_fast(rng, want["info:legal_action_mask"])
        want = orc.step(a)
        a_pool.step(a)
    b_pool = capi.CPool(game, n, seed=99)
    b_pool.state_import(a_pool.state_export())
    for t in range(40):
        a = policy(game, rng, want["info:legal_action_mask"], legal_share=0.8)
        want = orc.step(a)
        assert_same(a_pool.step(a), want, f"source step {t}")
        assert_same(b_pool.step(a), want, f"imported step {t}")


@pytest.mark.parametrize("game", GAMES)
def test_300000_envs_on_the_128_thread_kernel(capi, game):
    import torch

    n = 300_000
    pool = capi.CPool(game, n, seed=13)
    orc = PgxOracle(game, n, seed=13)
    rng = np.random.default_rng(6)
    pool.reset_device()
    want = orc.reset()
    assert_same(torch_out(pool), want, "reset")
    for t in range(30):
        a = policy(game, rng, want["info:legal_action_mask"], legal_share=0.0) if t % 3 == 0 \
            else legal_fast(rng, want["info:legal_action_mask"])
        pool.step_device(torch.from_numpy(a).cuda())
        want = orc.step(a)
        assert_same(torch_out(pool), want, f"step {t}")


_BLOCK_BODY = r"""
import sys
import numpy as np
import torch
sys.path[:0] = [{root!r}, {tests!r}]
from envpool_b200 import _capi
from test_gpu_pgx import PgxOracle, assert_same, legal_fast, policy, torch_out
for game in ("TicTacToe", "ConnectFour"):
    for n in (1, 255, 70001):
        pool = _capi.CPool(game, n, seed=17)
        orc = PgxOracle(game, n, seed=17)
        rng = np.random.default_rng(n)
        pool.reset_device()
        want = orc.reset()
        assert_same(torch_out(pool), want, "reset")
        for t in range(25):
            a = policy(game, rng, want["info:legal_action_mask"], legal_share=0.0) if t % 4 == 0 \
                else legal_fast(rng, want["info:legal_action_mask"])
            pool.step_device(torch.from_numpy(a).cuda())
            want = orc.step(a)
            assert_same(torch_out(pool), want, f"{{game}} n={{n}} step {{t}}")
print("ok")
"""


@pytest.mark.parametrize("block", [64])
def test_forced_step_kernel_block(block):
    """ENVPOOL_B200_STEP_BLOCK is read once per process: the 64-thread step kernel runs in a
    subprocess of its own, at batch sizes that leave a partial last CTA."""
    root = os.path.dirname(HERE)
    env = dict(os.environ, ENVPOOL_B200_STEP_BLOCK=str(block))
    r = subprocess.run([sys.executable, "-c", _BLOCK_BODY.format(root=root, tests=HERE)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


# ---------------------------------------------------------------------------- peer exchange
from exchange_cases import PgxKind, Ranks  # noqa: E402


@pytest.mark.parametrize("game", GAMES)
def test_exchange(game):
    """Direct exchanged steps (push_kernel forwards both player rows behind the step kernel)
    byte for byte against the un-exchanged twins, and the twins against the oracle."""
    import torch

    n, W = 1001, 2
    with Ranks(PgxKind(game, game), n, W) as x:
        x.attach()
        x.reset()
        x.steps_direct(20)
        # the twins against the oracle: global env g of rank r has seed + g
        orc = PgxOracle(game, W * n, seed=x.seed, env_seed=np.arange(W * n) + x.seed)
        orc.reset()
        for t in range(20):
            want = orc.step(x.acts[t % x.T])
        got = {}
        for k in x.twins[0].keys:
            got[k.name] = np.concatenate([tw.outputs_torch()[k.name].cpu().numpy()
                                          for tw in x.twins])
        assert_same(got, want, f"{game} exchanged twins vs oracle")
        torch.cuda.synchronize()


# ---------------------------------------------------------------------------- pool layouts
sys.path[:0] = [GOLDEN, os.path.join(GOLDEN, "pgx")]
from make_pgx_pool_layouts import FIXTURE as LAYOUTS, cases as layout_cases  # noqa: E402
from make_pool_layouts import describe  # noqa: E402


@pytest.mark.parametrize("case", sorted(dict(layout_cases(pgx_lib.GAMES))))
def test_pool_layout(capi, case):
    """Keys (per-player columns with their leading player dimension), slab size, state blob
    layout, bytes_per_env_step and launch count of every TicTacToe / ConnectFour pool against
    tests/golden/pgx/pool_layouts.json."""
    with open(LAYOUTS) as f:
        want = json.load(f)[case]
    assert describe(capi, *dict(layout_cases(pgx_lib.GAMES))[case]) == want
