"""GPU: PGX Go9x9-v1, Go13x13-v1 and Go19x19-v1 bit for bit against the C restatement
(oracle/go_oracle.c), the reference's own thread pool (oracle/_ref/libgo_ref.so, when build()
made it), the fixtures recorded from it (tests/golden/pgx/go/) and the scripts of
pgx_go_scripts.py, through every entry point: the host path (sync, async, permuted and partial
batches), make_gymnasium / make_dm, the pybind `_send` with explicit players.env_id rows,
step_device, the step chains (graph and direct), the timed chain, the fused rollout at T = 7,
snapshots, large pools, the peer exchange and the pool layouts.  The helpers are test_gpu_pgx.py's
and test_pgx_go.py's."""
import glob
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from test_gpu_pgx import assert_same, flat_ref, legal_fast, torch_out
from test_pgx_go import FIXTURE_DIR, load_fixture, pool_kwargs, row
from pgx_go_scripts import scripts

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import go_lib  # noqa: E402
from oracle.go_lib import GAMES, actions, first_player_actions  # noqa: E402
from oracle.go_lib import GoOracle as Oracle, GoRef as Ref  # noqa: E402

pytestmark = pytest.mark.gpu
FIXTURES = sorted(glob.glob(os.path.join(FIXTURE_DIR, "*.npz")))
TASK_ID = {g: f"{g}-v1" for g in GAMES}
I32 = np.iinfo(np.int32)


def policy(game, rng, mask, legal_share=0.9):
    """A legal action with probability legal_share, else any of -1..S^2+1 or INT_MIN / INT_MAX."""
    n = mask.shape[0]
    a = legal_fast(rng, mask).astype(np.int64)
    u = rng.random(n)
    a = np.where(u >= legal_share, rng.integers(-1, actions(game) + 1, n), a)
    a = np.where(u > 0.995, np.where(rng.random(n) < 0.5, I32.min, I32.max), a)
    return a.astype(np.int32)


def no_pass(mask):
    """The mask without the pass unless it is the only legal action (games run to their limit)."""
    m = mask.copy()
    m[:, -1] = ~m[:, :-1].any(1)
    return m


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_host_path(capi, path):
    meta, data = load_fixture(path)
    pool = capi.CPool(meta["game"], meta["num_envs"], seed=meta["seed"], **pool_kwargs(meta))
    assert_same(pool.reset(), row(data, 0), "reset")
    for t, a in enumerate(data["action"]):
        assert_same(pool.step(a), row(data, t + 1), f"step {t}")


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_gymnasium_and_dm(path):
    import envpool_b200

    meta, data = load_fixture(path)
    task, n = TASK_ID[meta["game"]], meta["num_envs"]
    kw = pool_kwargs(meta)
    gym = envpool_b200.make_gymnasium(task, num_envs=n, seed=meta["seed"], **kw)
    dm = envpool_b200.make_dm(task, num_envs=n, seed=meta["seed"], **kw)
    obs, info = gym.reset()
    ts = dm.reset()
    assert np.array_equal(obs, data["obs"][0]) and np.array_equal(ts.observation.obs, data["obs"][0])
    for t, a in enumerate(data["action"]):
        obs, rew, term, trunc, info = gym.step(a)
        ts = dm.step(a)
        w = row(data, t + 1)
        if "obs" in w:
            assert np.array_equal(obs, w["obs"]) and np.array_equal(ts.observation.obs, w["obs"]), t
        assert np.array_equal(rew, w["reward"]) and np.array_equal(ts.reward, w["reward"]), t
        assert np.array_equal(term | trunc, w["done"]) and not trunc.any(), t
        for k in ("board", "current_player", "legal_action_mask", "ko", "is_psk",
                  "consecutive_pass_count", "black_area", "white_area"):
            assert np.array_equal(info[k], w["info:" + k]), (t, k)
        assert np.array_equal(info["players"]["id"], w["info:players.id"]), t
        assert np.array_equal(ts.discount, w["discount"]) and np.array_equal(ts.step_type, w["step_type"])


@pytest.mark.parametrize("game", list(GAMES))
def test_scripts_host_and_device(capi, game):
    import torch

    sc = list(scripts(game).values())
    n = len(sc)
    orc = Oracle(game, n, seed=2)
    host, dev = capi.CPool(game, n, seed=2), capi.CPool(game, n, seed=2)
    want = orc.reset()
    assert_same(host.reset(), want, "host reset")
    dev.reset_device()
    assert_same(torch_out(dev), want, "device reset")
    for t in range(max(len(s) for s in sc) + 3):
        mask = want["info:legal_action_mask"]
        a = np.array([s[t] if t < len(s) else int(np.argmax(mask[i])) for i, s in enumerate(sc)],
                     np.int32)
        want = orc.step(a)
        assert_same(host.step(a), want, f"host step {t}")
        dev.step_device(torch.from_numpy(a).cuda())
        assert_same(torch_out(dev), want, f"step_device {t}")


@pytest.mark.parametrize("game,n", [("Go9x9", 256), ("Go13x13", 64), ("Go19x19", 32)])
def test_legal_play_to_max_terminal_steps(capi, game, n):
    """Legal play without passes until every game ends on the step limit or earlier: the whole
    hash history is written and scanned."""
    A = actions(game) - 1
    pool = capi.CPool(game, n, seed=9)
    orc = Oracle(game, n, seed=9)
    ref = Ref(game, n, seed=9) if go_lib.ref_available() else None
    want = orc.reset()
    assert_same(pool.reset(), want, "reset")
    if ref is not None:
        assert_same(flat_ref(ref.reset()), want, "ref reset")
    rng = np.random.default_rng(1)
    limit = 0
    for t in range(2 * A + 2):
        a = legal_fast(rng, no_pass(want["info:legal_action_mask"]))
        want = orc.step(a)
        assert_same(pool.step(a), want, f"step {t}")
        if ref is not None:
            assert_same(flat_ref(ref.step(a)), want, f"ref step {t}")
        limit += int((want["done"] & (want["elapsed_step"] == 2 * A)).sum())
    assert limit > 0


@pytest.mark.parametrize("game", list(GAMES))
def test_every_entry_point_gives_the_same_outputs_and_state(capi, game):
    """The host path, step_device, graph and direct chains, the timed chain and the fused
    rollout at T = 7 (the last rollout shorter) leave the same outputs and state blob."""
    import torch

    n, T, K = {"Go9x9": 600, "Go13x13": 200, "Go19x19": 100}[game], 7, 40
    rng = np.random.default_rng(5)
    orc = Oracle(game, n, seed=11, komi=0.5, max_terminal_steps=30)
    want = [orc.reset()]
    acts = np.empty((K, n), np.int32)
    for k in range(K):
        acts[k] = policy(game, rng, want[-1]["info:legal_action_mask"], 0.97)
        want.append(orc.step(acts[k]))
    d_acts = torch.from_numpy(acts).cuda()

    def fresh():
        p = capi.CPool(game, n, seed=11, komi=0.5, max_terminal_steps=30)
        p.reset_device()
        return p

    blobs = {}
    p = capi.CPool(game, n, seed=11, komi=0.5, max_terminal_steps=30)
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


@pytest.mark.parametrize("game", list(GAMES))
def test_async_permuted_and_partial_batches(capi, game):
    PER = ("info:players.env_id", "reward", "discount", "obs", "info:players.id")
    n, B = 200, 50
    rng = np.random.default_rng(9)
    pool = capi.CPool(game, n, seed=3, batch_size=B)
    orc = Oracle(game, n, seed=3)
    pool.reset_async()
    want = orc.reset()
    for b in range(n // B):
        assert_same(pool.recv(), {k: v[b * B * (2 if k in PER else 1):
                                        (b + 1) * B * (2 if k in PER else 1)]
                                  for k, v in want.items()}, f"async reset batch {b}")
    mask = want["info:legal_action_mask"].copy()
    for t in range(60):
        ids = rng.permutation(n).astype(np.int32)[:B]
        a = policy(game, rng, mask[ids])
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
        a = policy(game, rng, mask[ids])
        w = orc.step(a, ids)
        assert_same(sync.step(a, ids), w, f"partial batch of {m}, step {t}")
        mask[ids] = w["info:legal_action_mask"]


@pytest.mark.parametrize("game", list(GAMES))
def test_explicit_players_env_id(game):
    """`_send([env_id, players.env_id, action])`: each env acts with its first player row."""
    import envpool_b200

    n = 32
    rng = np.random.default_rng(2)
    env = envpool_b200.make_gymnasium(TASK_ID[game], num_envs=n, seed=5)
    orc = Oracle(game, n, seed=5)
    env.reset()
    want = orc.reset()
    ids = np.arange(n, dtype=np.int32)
    for t in range(60):
        pids = np.concatenate([ids, ids[rng.integers(0, n, size=n // 2)]])
        pids = pids[rng.permutation(len(pids))].astype(np.int32)
        acts = policy(game, rng, want["info:legal_action_mask"][pids])
        want = orc.step(first_player_actions(ids, pids, acts))
        env._send([ids, pids, acts])
        for k, g in zip(env._state_keys, env._recv()):
            assert np.array_equal(g, want[k]), (t, k)


@pytest.mark.parametrize("game", list(GAMES))
def test_snapshot_continues_in_a_pool_with_another_seed(capi, game):
    """The blob carries komi and max_terminal_steps: the imported pool, built with neither,
    scores the games that end on the 20-step limit as the source does."""
    n = 77
    rng = np.random.default_rng(4)
    a_pool = capi.CPool(game, n, seed=21, komi=-3.5, max_terminal_steps=20)
    orc = Oracle(game, n, seed=21, komi=-3.5, max_terminal_steps=20)
    want = orc.reset()
    a_pool.reset()
    for _ in range(9):
        a = legal_fast(rng, want["info:legal_action_mask"])
        want = orc.step(a)
        a_pool.step(a)
    b_pool = capi.CPool(game, n, seed=99)
    b_pool.state_import(a_pool.state_export())
    with pytest.raises(capi.EpbError, match="state import"):
        b_pool.go_config(7.5, 0)  # the imported configuration stays
    limit_ends = 0
    for t in range(40):
        a = policy(game, rng, want["info:legal_action_mask"], 0.98)
        want = orc.step(a)
        assert_same(a_pool.step(a), want, f"source step {t}")
        assert_same(b_pool.step(a), want, f"imported step {t}")
        limit_ends += int((want["done"] & (want["elapsed_step"] == 20) &
                           (want["reward"].reshape(n, 2) != 0).all(1)).sum())
    assert limit_ends > 0


@pytest.mark.parametrize("game,n", [("Go9x9", 65536), ("Go19x19", 16384)])
def test_large_pool_sampled_rows(capi, game, n):
    import torch

    ids = np.unique(np.concatenate([np.arange(64), np.arange(n - 64, n),
                                    np.arange(0, n, 997)])).astype(np.int32)
    pool = capi.CPool(game, n, seed=13)
    orc = Oracle(game, len(ids), seed=13, env_seed=13 + ids)
    rng = np.random.default_rng(6)
    pool.reset_device()
    want = orc.reset()
    acts = np.zeros(n, np.int32)

    def pick(out):  # the sampled rows; the id columns count the oracle's rows 0, 1, ...
        return {k: v[ids] for k, v in out.items() if k not in ("info:env_id", "info:players.env_id")}

    assert_same(pick(torch_out(pool)), {k: v for k, v in want.items()
                                        if k not in ("info:env_id", "info:players.env_id")}, "reset")
    for t in range(12):
        a = policy(game, rng, want["info:legal_action_mask"], 0.98)
        acts[:] = rng.integers(0, actions(game), n)
        acts[ids] = a
        pool.step_device(torch.from_numpy(acts).cuda())
        want = orc.step(a)
        got = torch_out(pool)
        assert np.array_equal(got["info:env_id"][ids], ids)
        assert_same(pick(got), {k: v for k, v in want.items()
                                if k not in ("info:env_id", "info:players.env_id")}, f"step {t}")


def test_make_gymnasium_plays_a_full_19x19_game():
    """make("Go19x19-v1", env_type="gymnasium") plays legal-random games to their end on the GPU
    with the reference's outputs (the oracle's where the reference is not built)."""
    import envpool_b200

    n = 8
    env = envpool_b200.make("Go19x19-v1", env_type="gymnasium", num_envs=n, max_num_players=2,
                            seed=31)
    chk = Ref("Go19x19", n, seed=31) if go_lib.ref_available() else Oracle("Go19x19", n, seed=31)
    obs, info = env.reset()
    chk.reset()
    rng = np.random.default_rng(8)
    ended = np.zeros(n, bool)
    for t in range(730):
        a = legal_fast(rng, no_pass(info["legal_action_mask"]))
        obs, rew, term, trunc, info = env.step(a)
        w = chk.step(a)
        assert np.array_equal(obs, w["obs"]) and np.array_equal(rew, w["reward"]), t
        assert np.array_equal(info["board"], w["info:board"]), t
        assert np.array_equal(info["legal_action_mask"], w["info:legal_action_mask"]), t
        ended |= term
        if ended.all():
            break
    assert ended.all()


def test_go_config_entry_point(capi):
    pool = capi.CPool("Go9x9", 4, seed=1)
    with pytest.raises(ValueError):
        pool.go_config(7.5, 163)
    with pytest.raises(ValueError):
        pool.go_config(7.5, -1)
    pool.go_config(0.0, 162)
    pool.reset()
    with pytest.raises(capi.EpbError, match="before the pool's first reset"):
        pool.go_config(7.5, 0)
    with pytest.raises(ValueError, match="not a Go pool"):
        capi.CPool("Hex", 4).go_config(7.5, 0)


from exchange_cases import PgxKind, Ranks  # noqa: E402


class GoKind(PgxKind):
    """exchange_cases' PGX kind with Go's action counts."""

    def actions(self, rng, shape):
        A = actions(self.task)
        a = rng.integers(-1, A + 1, size=shape)
        return np.where(rng.random(shape) < 0.97, rng.integers(0, A, size=shape), a).astype(np.int32)


@pytest.mark.parametrize("game", list(GAMES))
def test_exchange(game):
    """Direct exchanged steps byte for byte against the un-exchanged twins, and the twins
    against the oracle."""
    import torch

    n, W = 101, 2
    with Ranks(GoKind(game, game), n, W) as x:
        x.attach()
        x.reset()
        x.steps_direct(12)
        orc = Oracle(game, W * n, seed=x.seed, env_seed=np.arange(W * n) + x.seed)
        orc.reset()
        for t in range(12):
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


@pytest.mark.parametrize("case", sorted(dict(layout_cases(GAMES))))
def test_pool_layout(capi, case):
    with open(os.path.join(FIXTURE_DIR, "pool_layouts.json")) as f:
        want = json.load(f)[case]
    assert describe(capi, *dict(layout_cases(GAMES))[case]) == want
