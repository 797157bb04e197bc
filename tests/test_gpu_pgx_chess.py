"""GPU: PGX Chess-v1 and GardnerChess-v1 bit for bit against the fixtures recorded from the
reference (tests/golden/pgx/chess/) and the C restatement (oracle/chess_oracle.c), which
test_pgx_chess.py holds to both, through every entry point: the scripts of pgx_chess_scripts.py,
the host path (sync, async, permuted and
partial batches), make_gymnasium / make_dm, the pybind `_send` with explicit players.env_id rows,
step_device, the step chains (graph and direct), the timed chain, the fused rollout at T = 7,
snapshots, perft on the device, pools whose obs column passes 2 GiB, the peer exchange and the
pool layouts.  Labels whose target lies
off the board are among the actions (the engine's rule for them is the oracle's)."""
import json
import os
import sys

import numpy as np
import pytest

from helpers import GOLDEN
from pgx_chess_scripts import scripts, seeds_with_both_orders
from test_gpu_pgx import assert_same, legal_fast, torch_out
from test_pgx_chess import FIXTURE_DIR, FIXTURES, PERFT, load_fixture, out_of_range, row

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import chess_lib  # noqa: E402
from oracle.chess_lib import GAMES, MAX_STEPS, actions, first_player_actions  # noqa: E402
from oracle.chess_lib import ChessOracle as Oracle  # noqa: E402

pytestmark = pytest.mark.gpu
TASK_ID = {g: f"{g}-v1" for g in GAMES}


def policy(game, rng, mask, legal_share=0.95):
    """A legal label with probability legal_share, else any in-range label (off-board targets
    included), else (1 in 8 of those) an out-of-range one."""
    n = mask.shape[0]
    a = legal_fast(rng, mask).astype(np.int64)
    u = rng.random(n)
    a = np.where(u >= legal_share, rng.integers(0, actions(game), n), a)
    a = np.where(u >= 1 - (1 - legal_share) / 8, out_of_range(game)[rng.integers(0, 6, n)], a)
    return a.astype(np.int32)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_host_path(capi, path):
    meta, data = load_fixture(path)
    pool = capi.CPool(meta["game"], meta["num_envs"], seed=meta["seed"])
    assert_same(pool.reset(), row(data, 0), "reset")
    for t, a in enumerate(data["action"]):
        assert_same(pool.step(a), row(data, t + 1), f"step {t}")


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_fixture_gymnasium_and_dm(path):
    import envpool_b200

    meta, data = load_fixture(path)
    task, n = TASK_ID[meta["game"]], meta["num_envs"]
    gym = envpool_b200.make_gymnasium(task, num_envs=n, seed=meta["seed"])
    dm = envpool_b200.make_dm(task, num_envs=n, seed=meta["seed"])
    obs, info = gym.reset()
    ts = dm.reset()
    assert np.array_equal(obs, data["obs"][0]) and np.array_equal(ts.observation.obs, data["obs"][0])
    names = [k for k, *_ in chess_lib.keys(meta["game"]) if k.startswith("info:") and
             "env_id" not in k and k != "info:players.id"]
    for t, a in enumerate(data["action"]):
        obs, rew, term, trunc, info = gym.step(a)
        ts = dm.step(a)
        w = row(data, t + 1)
        if "obs" in w:
            assert np.array_equal(obs, w["obs"]) and np.array_equal(ts.observation.obs, w["obs"]), t
        assert np.array_equal(rew, w["reward"]) and np.array_equal(ts.reward, w["reward"]), t
        assert np.array_equal(term | trunc, w["done"]) and not trunc.any(), t
        for k in names:
            assert np.array_equal(info[k[5:]], w[k]), (t, k)
        assert np.array_equal(ts.discount, w["discount"]) and np.array_equal(ts.step_type, w["step_type"])


@pytest.mark.parametrize("game", list(GAMES))
def test_scripts_host_and_device(capi, game):
    """Every script, the off-board ones included, under both player orders."""
    import torch

    sc = list(scripts(game).values()) * 2
    n = len(sc)
    s0, s1 = seeds_with_both_orders()
    seeds = np.array([s0] * (n // 2) + [s1] * (n // 2), np.int32)
    orc = Oracle(game, n, env_seed=seeds)
    host = capi.CPool(game, n, env_seed=seeds)
    dev = capi.CPool(game, n, env_seed=seeds)
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


@pytest.mark.parametrize("game", list(GAMES))
def test_legal_play_to_the_step_limit(capi, game):
    """Legal-random games run to their ends, the step limit included (11 Chess and 1 GardnerChess
    game of these 256 reach it): every stored key is written and scanned.  The oracle holds the
    reference's outputs over these same games (test_pgx_chess.py)."""
    n = 256
    pool = capi.CPool(game, n, seed=9)
    orc = Oracle(game, n, seed=9)
    want = orc.reset()
    assert_same(pool.reset(), want, "reset")
    rng = np.random.default_rng(1)
    limit = 0
    for t in range(MAX_STEPS[game] + 2):
        a = legal_fast(rng, want["info:legal_action_mask"])
        want = orc.step(a)
        assert_same(pool.step(a), want, f"step {t}")
        limit += int((want["done"] & (want["elapsed_step"] == MAX_STEPS[game])).sum())
    assert limit > 0


@pytest.mark.parametrize("game", list(GAMES))
def test_random_labels_host_and_device(capi, game):
    """Every kind of label, off-board targets and out-of-range values included, through the host
    path and step_device."""
    import torch

    n = 300
    rng = np.random.default_rng(2)
    orc = Oracle(game, n, seed=2)
    host, dev = capi.CPool(game, n, seed=2), capi.CPool(game, n, seed=2)
    want = orc.reset()
    assert_same(host.reset(), want, "host reset")
    dev.reset_device()
    assert_same(torch_out(dev), want, "device reset")
    for t in range(150):
        a = policy(game, rng, want["info:legal_action_mask"], 0.9)
        want = orc.step(a)
        assert_same(host.step(a), want, f"host step {t}")
        dev.step_device(torch.from_numpy(a).cuda())
        assert_same(torch_out(dev), want, f"step_device {t}")


@pytest.mark.parametrize("game", list(GAMES))
def test_gymnasium_and_dm(game):
    import envpool_b200

    n = 16
    rng = np.random.default_rng(3)
    gym = envpool_b200.make_gymnasium(TASK_ID[game], num_envs=n, seed=4)
    dm = envpool_b200.make_dm(TASK_ID[game], num_envs=n, seed=4)
    orc = Oracle(game, n, seed=4)
    obs, info = gym.reset()
    ts = dm.reset()
    want = orc.reset()
    assert np.array_equal(obs, want["obs"]) and np.array_equal(ts.observation.obs, want["obs"])
    names = [k for k, *_ in chess_lib.keys(game) if k.startswith("info:") and "env_id" not in k
             and k != "info:players.id"]
    for t in range(120):
        a = policy(game, rng, want["info:legal_action_mask"], 0.97)
        want = orc.step(a)
        obs, rew, term, trunc, info = gym.step(a)
        ts = dm.step(a)
        assert np.array_equal(obs, want["obs"]) and np.array_equal(ts.observation.obs, want["obs"]), t
        assert np.array_equal(rew, want["reward"]) and np.array_equal(ts.reward, want["reward"]), t
        assert np.array_equal(term | trunc, want["done"]) and not trunc.any(), t
        for k in names:
            assert np.array_equal(info[k[5:]], want[k]), (t, k)
        assert np.array_equal(ts.discount, want["discount"])
        assert np.array_equal(ts.step_type, want["step_type"])


@pytest.mark.parametrize("game", list(GAMES))
def test_every_entry_point_gives_the_same_outputs_and_state(capi, game):
    """The host path, step_device, graph and direct chains, the timed chain and the fused
    rollout at T = 7 (the last rollout shorter) leave the same outputs and state blob."""
    import torch

    n, T, K = 300, 7, 40
    rng = np.random.default_rng(5)
    orc = Oracle(game, n, seed=11)
    want = [orc.reset()]
    acts = np.empty((K, n), np.int32)
    for k in range(K):
        acts[k] = policy(game, rng, want[-1]["info:legal_action_mask"], 0.97)
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
    n = 77
    rng = np.random.default_rng(4)
    a_pool = capi.CPool(game, n, seed=21)
    orc = Oracle(game, n, seed=21)
    want = orc.reset()
    a_pool.reset()
    for _ in range(30):
        a = legal_fast(rng, want["info:legal_action_mask"])
        want = orc.step(a)
        a_pool.step(a)
    b_pool = capi.CPool(game, n, seed=99)
    b_pool.state_import(a_pool.state_export())
    for t in range(60):
        a = policy(game, rng, want["info:legal_action_mask"], 0.98)
        want = orc.step(a)
        assert_same(a_pool.step(a), want, f"source step {t}")
        assert_same(b_pool.step(a), want, f"imported step {t}")


def test_perft_on_the_device(capi):
    """perft(d + 1) from the initial position through step_device, d = 0..3: every ply-d position
    reached by its move sequence, the masks of the envs not done summed."""
    import torch

    seqs = np.zeros((1, 0), np.int32)
    for d in range(4):
        n = len(seqs)
        pool = capi.CPool("Chess", n, seed=1)
        pool.reset_device()
        for k in range(d):
            pool.step_device(torch.from_numpy(np.ascontiguousarray(seqs[:, k])).cuda())
        out = pool.outputs_torch()
        mask = (out["info:legal_action_mask"] & ~out["done"][:, None]).cpu().numpy()
        assert int(mask.sum()) == PERFT[d], d
        e, a = np.nonzero(mask)
        seqs = np.concatenate([seqs[e], a[:, None].astype(np.int32)], 1)
    assert len(seqs) == PERFT[3]


@pytest.mark.parametrize("game,n", [("Chess", 40000), ("GardnerChess", 100000)])
def test_large_pool_sampled_rows(capi, game, n):
    """Pools whose obs column passes 2 GiB (Chess: 40000 x 60928 bytes, GardnerChess: 100000 x
    23000): rows at both ends of every column through step_device and the captured chain.  The
    rows are picked on the device, so no whole column is copied to the host.  Cost: a pool pins
    one host mirror of its output slab when it is created (epb_create, at least one slab even
    past the 1 GiB budget for pinned slabs), 2.64 GB here for Chess and 2.44 GB for
    GardnerChess, beside as much device memory plus the state; the test holds one such pool at a
    time and closes it before returning, so its peak is one slab of pinned host memory."""
    import torch

    ids = np.unique(np.concatenate([np.arange(32), np.arange(n - 32, n),
                                    np.arange(0, n, 4999)])).astype(np.int32)
    d_ids = torch.from_numpy(ids).long().cuda()
    pool = capi.CPool(game, n, seed=13)
    assert pool.outputs_torch()["obs"].numel() * 4 > 2 ** 31
    orc = Oracle(game, len(ids), seed=13, env_seed=13 + ids)
    rng = np.random.default_rng(6)
    skip = ("info:env_id", "info:players.env_id")

    def pick():
        got = {}
        for k, v in pool.outputs_torch().items():
            if k in skip:
                continue
            got[k] = v[d_ids].cpu().numpy()
        return got

    pool.reset_device()
    want = orc.reset()
    assert_same(pick(), {k: v for k, v in want.items() if k not in skip}, "reset")
    assert np.array_equal(pool.outputs_torch()["info:env_id"][d_ids].cpu().numpy(), ids)
    acts = np.zeros(n, np.int32)
    for t in range(6):
        a = policy(game, rng, want["info:legal_action_mask"], 0.98)
        acts[:] = rng.integers(0, actions(game), n)
        acts[ids] = a
        pool.step_device(torch.from_numpy(acts).cuda())
        want = orc.step(a)
        assert_same(pick(), {k: v for k, v in want.items() if k not in skip}, f"step {t}")
    K = 4
    chain = np.empty((K, n), np.int32)
    for k in range(K):
        a = policy(game, rng, want["info:legal_action_mask"], 0.98)
        chain[k] = rng.integers(0, actions(game), n)
        chain[k, ids] = a
        want = orc.step(a)
    pool.step_many_device(torch.from_numpy(chain).cuda(), 0, K, use_graph=True)
    torch.cuda.synchronize()
    assert_same(pick(), {k: v for k, v in want.items() if k not in skip}, "captured chain")
    pool.close()
    torch.cuda.empty_cache()


from exchange_cases import PgxKind, Ranks  # noqa: E402


class ChessKind(PgxKind):
    """exchange_cases' PGX kind with the chess games' label counts (off-board targets and
    out-of-range values among them)."""

    def actions(self, rng, shape):
        A = actions(self.task)
        a = rng.integers(-1, A + 1, size=shape)
        return np.where(rng.random(shape) < 0.97, rng.integers(0, A, size=shape), a).astype(np.int32)


@pytest.mark.parametrize("game", list(GAMES))
def test_exchange(game):
    """Direct exchanged steps byte for byte against the un-exchanged twins, and the twins against
    the oracle: Chess's env keys 5..9 travel beside OutView (LaunchArgs::env_hi)."""
    import torch

    n, W = 101, 2
    with Ranks(ChessKind(game, game), n, W) as x:
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
