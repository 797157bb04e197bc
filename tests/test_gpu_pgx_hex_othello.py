"""GPU: PGX Hex-v1 and Othello-v1 bit for bit against the C restatement (oracle/hex_othello_oracle.c), the
reference's own thread pool (oracle/_ref/libhex_othello_ref.so, when build() made it), the fixtures recorded from it
(tests/golden/pgx/hex_othello/) and the scripts of the seeded search
(pgx_hex_othello_scripts.py), through every entry point: the host path (sync, async, permuted
and partial batches), make_gymnasium / make_dm, the pybind `_send` with explicit
players.env_id rows, step_device, the step chains (graph and direct), the timed chain, the
fused rollout at an odd T, snapshots, the 64- and 128-thread step kernels, the peer exchange and
the pool layouts.  The helpers are test_gpu_pgx.py's; the checkers are oracle/hex_othello_lib.py's."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import GOLDEN
import test_gpu_pgx as base
from test_gpu_pgx import assert_same, flat_ref, legal_fast, load_fixture, policy, torch_out
from pgx_hex_othello_scripts import scripts

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import hex_othello_lib  # noqa: E402
from oracle.hex_othello_lib import ACTIONS, first_player_actions  # noqa: E402
from oracle.hex_othello_lib import HexOthelloOracle as Oracle, HexOthelloRef as Ref  # noqa: E402

pytestmark = pytest.mark.gpu
GAMES = ["Hex", "Othello"]
TASK_ID = {"Hex": "Hex-v1", "Othello": "Othello-v1"}
FIXTURE_DIR = os.path.join(GOLDEN, "pgx", "hex_othello")
FIXTURES = sorted(glob.glob(os.path.join(FIXTURE_DIR, "*.npz")))


@pytest.mark.parametrize("game", GAMES)
def test_random_and_legal_play_against_oracle_and_ref(capi, game):
    n, T = 2048, 1000
    pool = capi.CPool(game, n, seed=7)
    orc = Oracle(game, n, seed=7)
    ref = Ref(game, n, seed=7) if hex_othello_lib.ref_available() else None
    want = orc.reset()
    assert_same(pool.reset(), want, f"{game} reset")
    if ref is not None:
        assert_same(flat_ref(ref.reset()), want, f"{game} ref reset")
    rng = np.random.default_rng(1)
    for t in range(T):
        mask = want["info:legal_action_mask"]
        a = legal_fast(rng, mask) if t % 4 else policy(game, rng, mask, legal_share=0.0)
        want = orc.step(a)
        assert_same(pool.step(a), want, f"{game} step {t}")
        if ref is not None:
            assert_same(flat_ref(ref.step(a)), want, f"{game} ref step {t}")


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_host_path(capi, path):
    base.test_fixture_host_path(capi, path)


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


def script_actions(game, out, t):
    """Step t of the search scripts, one env each; an env past its script plays legally."""
    acts = list(scripts(game).values())
    mask = out["info:legal_action_mask"]
    return np.array([s[t] if t < len(s) else int(np.argmax(mask[i])) for i, s in enumerate(acts)],
                    np.int32), max(len(s) for s in acts) + 3


@pytest.mark.parametrize("game", GAMES)
def test_search_scripts_host_and_device(capi, game):
    """Every class the search reached, through the host path and step_device."""
    import torch

    n = len(scripts(game))
    orc = Oracle(game, n, seed=2)
    host, dev = capi.CPool(game, n, seed=2), capi.CPool(game, n, seed=2)
    want = orc.reset()
    assert_same(host.reset(), want, "host reset")
    dev.reset_device()
    assert_same(torch_out(dev), want, "device reset")
    _, T = script_actions(game, want, 0)
    for t in range(T):
        a, _ = script_actions(game, want, t)
        want = orc.step(a)
        assert_same(host.step(a), want, f"host step {t}")
        dev.step_device(torch.from_numpy(a).cuda())
        assert_same(torch_out(dev), want, f"step_device {t}")


@pytest.mark.parametrize("game", GAMES)
def test_max_num_players_must_be_two(game):
    import envpool_b200

    for players in (1, 3):
        with pytest.raises(ValueError, match="max_num_players must be 2"):
            envpool_b200.make_gymnasium(TASK_ID[game], num_envs=4, max_num_players=players)


@pytest.mark.parametrize("game", GAMES)
def test_every_entry_point_gives_the_same_outputs_and_state(capi, game):
    """The host path, step_device, graph and direct chains, the timed chain and the fused
    rollout at T = 7 (odd, the last rollout shorter) leave the same outputs and state blob."""
    import torch

    n, T, K = 3000, 7, 40
    rng = np.random.default_rng(5)
    orc = Oracle(game, n, seed=11)
    want = [orc.reset()]
    acts = np.empty((K, n), np.int32)
    for k in range(K):
        m = want[-1]["info:legal_action_mask"]
        acts[k] = np.where(rng.random(n) < 0.95, legal_fast(rng, m),
                           policy(game, rng, m, legal_share=0.0))
        want.append(orc.step(acts[k]))
    d_acts = torch.from_numpy(acts).cuda()

    def fresh():
        p = capi.CPool(game, n, seed=11)
        p.reset_device()
        return p

    blobs = {}
    p = capi.CPool(game, n, seed=11)
    assert_same(p.reset(), want[0], "host reset")
    for k in range(K):
        assert_same(p.step(acts[k]), want[k + 1], f"host step {k}")
    blobs["host"] = p.state_export()
    p = fresh()
    for k in range(K):
        p.step_device(d_acts[k])
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
    for r in range((K + T - 1) // T):
        steps = min(T, K - r * T)
        p.rollout_device(d_acts[r * T:r * T + steps].contiguous(), steps, cols)
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
    orc = Oracle(game, n, seed=3)
    pool.reset_async()
    want = orc.reset()
    for b in range(n // B):
        assert_same(pool.recv(), {k: v[b * B * (2 if k in base.PER_PLAYER else 1):
                                        (b + 1) * B * (2 if k in base.PER_PLAYER else 1)]
                                  for k, v in want.items()}, f"async reset batch {b}")
    mask = want["info:legal_action_mask"].copy()
    for t in range(60):
        ids = rng.permutation(n).astype(np.int32)[:B]
        a = policy(game, rng, mask[ids], legal_share=0.9)
        pool.send(a, ids)
        w = orc.step(a, ids)
        assert_same(pool.recv(), w, f"async permuted step {t}")
        mask[ids] = w["info:legal_action_mask"]
    sync = capi.CPool(game, n, seed=4)
    orc = Oracle(game, n, seed=4)
    want = orc.reset()
    assert_same(sync.reset(), want, "sync reset")
    mask = want["info:legal_action_mask"].copy()
    for t in range(60):
        m = int(rng.integers(1, n + 1))
        ids = rng.permutation(n).astype(np.int32)[:m]
        a = policy(game, rng, mask[ids], legal_share=0.9)
        w = orc.step(a, ids)
        assert_same(sync.step(a, ids), w, f"partial batch of {m}, step {t}")
        mask[ids] = w["info:legal_action_mask"]


@pytest.mark.parametrize("game", GAMES)
def test_explicit_players_env_id(game):
    """`_send([env_id, players.env_id, action])`: each env acts with its first player row."""
    import envpool_b200

    n = 64
    rng = np.random.default_rng(2)
    env = envpool_b200.make_gymnasium(TASK_ID[game], num_envs=n, seed=5)
    orc = Oracle(game, n, seed=5)
    ref = Ref(game, n, seed=5) if hex_othello_lib.ref_available() else None
    env.reset()
    want = orc.reset()
    if ref is not None:
        ref.reset()
    ids = np.arange(n, dtype=np.int32)
    for t in range(80):
        pids = np.concatenate([ids, ids[rng.integers(0, n, size=n // 2)]])
        pids = pids[rng.permutation(len(pids))].astype(np.int32)
        acts = policy(game, rng, want["info:legal_action_mask"][pids], legal_share=0.9)
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


@pytest.mark.parametrize("game", GAMES)
def test_snapshot_continues_in_a_pool_with_another_seed(capi, game):
    n = 777
    rng = np.random.default_rng(4)
    a_pool = capi.CPool(game, n, seed=21)
    orc = Oracle(game, n, seed=21)
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
    orc = Oracle(game, n, seed=13)
    rng = np.random.default_rng(6)
    pool.reset_device()
    want = orc.reset()
    assert_same(torch_out(pool), want, "reset")
    for t in range(30):
        a = policy(game, rng, want["info:legal_action_mask"], legal_share=0.0) if t % 5 == 0 \
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
from test_gpu_pgx import assert_same, legal_fast, policy, torch_out
from oracle.hex_othello_lib import HexOthelloOracle as Oracle
for game in ("Hex", "Othello"):
    for n in (1, 255, 70001):
        pool = _capi.CPool(game, n, seed=17)
        orc = Oracle(game, n, seed=17)
        rng = np.random.default_rng(n)
        pool.reset_device()
        want = orc.reset()
        assert_same(torch_out(pool), want, "reset")
        for t in range(25):
            a = policy(game, rng, want["info:legal_action_mask"], legal_share=0.0) if t % 6 == 0 \
                else legal_fast(rng, want["info:legal_action_mask"])
            pool.step_device(torch.from_numpy(a).cuda())
            want = orc.step(a)
            assert_same(torch_out(pool), want, f"{{game}} n={{n}} step {{t}}")
print("ok")
"""


def test_forced_64_thread_step_kernel():
    """ENVPOOL_B200_STEP_BLOCK is read once per process: the 64-thread kernel in a subprocess."""
    root = os.path.dirname(HERE)
    env = dict(os.environ, ENVPOOL_B200_STEP_BLOCK="64")
    r = subprocess.run([sys.executable, "-c", _BLOCK_BODY.format(root=root, tests=HERE)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


from exchange_cases import PgxKind, Ranks  # noqa: E402


class HexOthelloKind(PgxKind):
    """exchange_cases' PGX kind with this module's action counts."""

    def actions(self, rng, shape):
        a = rng.integers(-1, ACTIONS[self.task] + 1, size=shape)
        return np.where(rng.random(shape) < 0.9,
                        rng.integers(0, ACTIONS[self.task], size=shape), a).astype(np.int32)


@pytest.mark.parametrize("game", GAMES)
def test_exchange(game):
    """Direct exchanged steps byte for byte against the un-exchanged twins, and the twins
    against the oracle."""
    import torch

    n, W = 1001, 2
    with Ranks(HexOthelloKind(game, game), n, W) as x:
        x.attach()
        x.reset()
        x.steps_direct(20)
        orc = Oracle(game, W * n, seed=x.seed, env_seed=np.arange(W * n) + x.seed)
        orc.reset()
        for t in range(20):
            want = orc.step(x.acts[t % x.T])
        got = {}
        for k in x.twins[0].keys:
            got[k.name] = np.concatenate([tw.outputs_torch()[k.name].cpu().numpy()
                                          for tw in x.twins])
        assert_same(got, want, f"{game} exchanged twins vs oracle")
        torch.cuda.synchronize()


sys.path[:0] = [GOLDEN, os.path.join(GOLDEN, "pgx")]
from make_pgx_pool_layouts import cases as layout_cases  # noqa: E402
from make_pool_layouts import describe  # noqa: E402


@pytest.mark.parametrize("case", sorted(dict(layout_cases(hex_othello_lib.GAMES))))
def test_pool_layout(capi, case):
    with open(os.path.join(FIXTURE_DIR, "pool_layouts.json")) as f:
        want = json.load(f)[case]
    assert describe(capi, *dict(layout_cases(hex_othello_lib.GAMES))[case]) == want
