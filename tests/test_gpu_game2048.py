"""GPU: Jumanji Game2048-v1 on the sm_90a kernel (envpool_b200/csrc/jumanji.cu), bit for bit
against the oracle (oracle/g2048_oracle.c), the reference's own thread pool (oracle/_ref, when the
build made it) and the fixtures recorded from it, through every entry point of the engine."""
import numpy as np
import pytest

from helpers import assert_batch_equal
from test_game2048 import (FIXTURES, RULE_ACTIONS, RULE_BOARD, cells, load_fixture, oracle_for,
                           rule_mask, rule_move)

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
# 3 replay boards and no initial board: every reset draws its random cell, the replay
# overwrites steps 1..3 and step 4 lands on an empty board, which ends the episode
SHORT_REPLAY = ",".join(str(v) for v in
                        [1, 1, 2, 2, 3, 4, 0, 0, 0, 2, 0, 0, 0, 5, 0, 0] +
                        [0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 3] +
                        [6, 5, 4, 3, 5, 4, 3, 2, 4, 3, 2, 1, 3, 2, 1, 1])
CONFIGS = {
    "default": dict(max_episode_steps=1000, add_random_cell=True, initial_board="",
                    replay_boards=""),
    "no_random_cell": dict(max_episode_steps=1000, add_random_cell=False,
                           initial_board="1,1,2,2,3,4,0,0,0,2,0,0,0,5,0,0", replay_boards=""),
    "replay_cycle": dict(max_episode_steps=3, add_random_cell=True, initial_board="",
                         replay_boards=SHORT_REPLAY),
}


def meta_for(config, n, seed):
    return dict(CONFIGS[config], num_envs=n, seed=seed)


def make_pool(capi, meta, **kw):
    pool = capi.CPool("Game2048", meta["num_envs"], seed=meta["seed"],
                      max_episode_steps=meta["max_episode_steps"],
                      iopt=1 if meta["add_random_cell"] else 0, **kw)
    ini, rep = cells(meta["initial_board"], 16), cells(meta["replay_boards"], 512)
    if ini is not None or rep is not None:
        pool.game2048_boards(ini, rep)
    return pool


def ref_for(meta):
    """The reference's own AsyncEnvPool<Game2048Env> when the build compiled it, else None."""
    from oracle import g2048_lib

    if not g2048_lib.ref_available():
        return None
    return g2048_lib.Game2048Ref(meta["num_envs"], seed=meta["seed"],
                                 max_episode_steps=meta["max_episode_steps"],
                                 add_random_cell=meta["add_random_cell"],
                                 initial_board=meta["initial_board"],
                                 replay_boards=meta["replay_boards"], num_threads=4)


def actions(rng, shape):
    """Directions 0..3, one in ten out of range (the env clamps them)."""
    a = rng.integers(0, 4, size=shape).astype(np.int64)
    odd = rng.random(shape) < 0.1
    a[odd] = rng.choice(np.array([-5, 4, INT32_MIN, INT32_MAX]), size=int(odd.sum()))
    return a.astype(np.int32)


def outputs(pool, n=None):
    return {k: v.cpu().numpy() for k, v in pool.outputs_torch(n).items()}


def eq(got, want, ctx):
    assert_batch_equal(got, want, "Game2048", 0.0, ctx)


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_random_rollouts_match_oracle_and_reference(capi, config):
    meta = meta_for(config, 2048, 21)
    pool, orc, ref = make_pool(capi, meta), oracle_for(meta), ref_for(meta)
    rng = np.random.default_rng(5)
    want = orc.reset()
    eq(pool.reset(), want, f"{config} reset")
    if ref is not None:
        eq(ref.reset(), want, f"{config} reference reset")
    for t in range(1000):
        a = actions(rng, 2048)
        want = orc.step(a)
        eq(pool.step(a), want, f"{config} t={t}")
        if ref is not None:
            eq(ref.step(a), want, f"{config} reference t={t}")


@pytest.mark.parametrize("name", FIXTURES)
def test_reference_fixtures_through_the_host_path(capi, name):
    meta, gold = load_fixture(name)
    pool = make_pool(capi, meta)
    keys = [k for k in gold if k != "actions"]
    eq(pool.reset(), {k: gold[k][0] for k in keys}, f"{name} reset")
    for t, a in enumerate(gold["actions"]):
        eq(pool.step(a), {k: gold[k][t + 1] for k in keys}, f"{name} t={t}")


def test_reference_rule_cases_through_make_gymnasium(capi):
    """The fixed six-move rollout from a configured board without random cells, and seeded
    determinism of reset boards (restated from the reference's own Game2048 tests)."""
    import envpool_b200 as ep

    env = ep.make_gymnasium("Game2048-v1", num_envs=1, seed=0, game2048_add_random_cell=False,
                            game2048_initial_board=",".join(map(str, RULE_BOARD.ravel())))
    board = RULE_BOARD.copy()
    obs, info = env.reset()
    np.testing.assert_array_equal(obs["board"][0], board)
    np.testing.assert_array_equal(obs["action_mask"][0], rule_mask(board))
    assert int(info["highest_tile"][0]) == 32
    for a in RULE_ACTIONS:
        board, reward = rule_move(board, a)
        obs, rew, term, trunc, info = env.step(np.array([a], np.int32))
        np.testing.assert_array_equal(obs["board"][0], board)
        np.testing.assert_array_equal(obs["action_mask"][0], rule_mask(board))
        assert float(rew[0]) == reward
        assert bool(term[0]) == (not rule_mask(board).any()) and not trunc[0]
        assert int(info["highest_tile"][0]) == 2 ** board.max()
    envs = [ep.make_gymnasium("Game2048-v1", num_envs=4, seed=7) for _ in range(2)]
    (o0, _), (o1, _) = envs[0].reset(), envs[1].reset()
    np.testing.assert_array_equal(o0["board"], o1["board"])
    np.testing.assert_array_equal(o0["action_mask"], o1["action_mask"])
    flat = o0["board"].reshape(4, 16)
    got = [(int(np.flatnonzero(b)[0]), int(b[np.flatnonzero(b)[0]])) for b in flat]
    assert got == [(12, 1), (15, 2), (8, 1), (0, 1)]


def test_make_gymnasium_and_make_dm_observations(capi):
    import envpool_b200 as ep

    env = ep.make_gymnasium("Game2048-v1", num_envs=8, seed=3)
    assert set(env.observation_space.keys()) == {"board", "action_mask"}
    obs, info = env.reset()
    assert isinstance(obs, dict) and set(obs) == {"board", "action_mask"}
    assert obs["board"].dtype == np.int32 and obs["board"].shape == (8, 4, 4)
    assert obs["action_mask"].dtype == np.bool_ and obs["action_mask"].shape == (8, 4)
    assert info["highest_tile"].dtype == np.int32 and info["highest_tile"].shape == (8,)
    obs, rew, term, trunc, info = env.step(np.zeros(8, np.int32))
    assert rew.dtype == np.float32 and term.dtype == np.bool_
    dm = ep.make_dm("Game2048-v1", num_envs=8, seed=3)
    ts = dm.reset()
    o = ts.observation
    assert type(o).__name__ == "State"
    assert list(o._fields) == ["env_id", "players", "board", "action_mask", "highest_tile"]
    assert o.board.dtype == np.int32 and o.board.shape == (8, 4, 4)
    assert o.action_mask.dtype == np.bool_ and o.highest_tile.dtype == np.int32
    ts = dm.step(np.zeros(8, np.int32))
    assert ts.observation.board.shape == (8, 4, 4)


@pytest.mark.parametrize("config", ["default", "replay_cycle"])
def test_every_entry_point_is_bit_identical(capi, config):
    """One action stream [T, N] through host step, step_device, step_many_device (graph and
    direct), step_many_timed and rollout_device in pieces.  Host step, step_device and the
    rollout are checked row by row against the oracle; every chain must leave the same last
    outputs and the same state blob."""
    import torch

    N, T = 3000, 96
    meta = meta_for(config, N, 31)
    rng = np.random.default_rng(7)
    acts = actions(rng, (T, N))
    d_acts = torch.from_numpy(acts).cuda()
    orc = oracle_for(meta)
    want0 = orc.reset()
    want = [orc.step(acts[t]) for t in range(T)]

    host = make_pool(capi, meta)
    eq(host.reset(), want0, "host reset")
    for t in range(T):
        eq(host.step(acts[t]), want[t], f"host t={t}")
    blob = host.state_export()

    dev = make_pool(capi, meta)
    dev.reset_device()
    torch.cuda.synchronize()
    eq(outputs(dev), want0, "device reset")
    for t in range(T):
        dev.step_device(d_acts[t])
        torch.cuda.synchronize()
        eq(outputs(dev), want[t], f"step_device t={t}")
    assert np.array_equal(dev.state_export(), blob)

    for how in ("graph", "direct", "timed"):
        p = make_pool(capi, meta)
        p.reset_device()
        if how == "timed":
            ms = p.step_many_timed(d_acts, 0, T, 8, T, use_graph=True)
            assert ms > 0
        else:
            p.step_many_device(d_acts, 0, T, use_graph=how == "graph")
        p.sync()
        eq(outputs(p), want[-1], f"{how} chain last step")
        assert np.array_equal(p.state_export(), blob), how

    roll = make_pool(capi, meta)
    roll.reset_device()
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.bool_): torch.bool}
    t0 = 0
    for piece in (1, 40, 55):
        cols = [torch.empty((piece, N) + k.shape, dtype=tdt[k.dtype], device="cuda")
                for k in roll.keys]
        roll.rollout_device(d_acts[t0:t0 + piece].contiguous(), piece, cols)
        roll.sync()
        for t in range(piece):
            got = {k.name: c[t].cpu().numpy() for k, c in zip(roll.keys, cols)}
            eq(got, want[t0 + t], f"rollout t={t0 + t}")
        t0 += piece
    assert np.array_equal(roll.state_export(), blob)


def test_async_send_recv_with_smaller_batches(capi):
    N, B = 1024, 256
    meta = meta_for("replay_cycle", N, 41)
    pool = make_pool(capi, meta, batch_size=B)
    orc = oracle_for(meta)
    rng = np.random.default_rng(3)
    pending = [orc.reset()]
    pool.reset_async()

    def take(rows):
        """The next `rows` rows the oracle says the engine hands out, in submission order."""
        out = {}
        while rows:
            head = pending[0]
            k = min(rows, len(head["info:env_id"]))
            for name, v in head.items():
                out.setdefault(name, []).append(v[:k])
            rest = {name: v[k:] for name, v in head.items()}
            if len(rest["info:env_id"]):
                pending[0] = rest
            else:
                pending.pop(0)
            rows -= k
        return {name: np.concatenate(v) for name, v in out.items()}

    for it in range(200):
        got = pool.recv()
        eq(got, take(B), f"async recv {it}")
        ids = got["info:env_id"]
        parts = (ids[: B // 2], ids[B // 2:]) if it % 5 == 2 else (ids,)
        for part in parts:
            a = actions(rng, len(part))
            pending.append(orc.step(a, part))
            pool.send(a, part)


def test_permuted_and_partial_batches_keep_other_envs(capi):
    N = 2000
    meta = meta_for("default", N, 51)
    pool, orc = make_pool(capi, meta), oracle_for(meta)
    rng = np.random.default_rng(11)
    eq(pool.reset(), orc.reset(), "reset")
    for t in range(300):
        if t % 3 == 0:
            ids = rng.permutation(N).astype(np.int32)
        else:
            ids = np.sort(rng.choice(N, size=int(rng.integers(1, N)), replace=False)).astype(
                np.int32)
            if t % 3 == 2:
                rng.shuffle(ids)
        before = pool.state_arrays(pool.state_export())
        before = {k: v.copy() for k, v in before.items()}
        a = actions(rng, len(ids))
        eq(pool.step(a, ids), orc.step(a, ids), f"t={t}")
        after = pool.state_arrays(pool.state_export())
        out = np.setdiff1d(np.arange(N), ids)
        for k in ("flags", "mt_idx", "istate", "mt"):
            b, c = before[k], after[k]
            sel = (slice(None), out) if k == "istate" else (
                (slice(None), out, slice(None)) if k == "mt" else out)
            assert np.array_equal(b[sel], c[sel]), (t, k)
        if t % 50 == 49:   # forced partial resets
            r = np.sort(rng.choice(N, size=300, replace=False)).astype(np.int32)
            eq(pool.reset(r), orc.reset(r), f"partial reset t={t}")


def test_snapshot_continues_in_a_pool_with_another_seed(capi):
    N = 1500
    meta = meta_for("default", N, 61)
    a, orc = make_pool(capi, meta), oracle_for(meta)
    rng = np.random.default_rng(13)
    eq(a.reset(), orc.reset(), "reset")
    for t in range(57):
        act = actions(rng, N)
        eq(a.step(act), orc.step(act), f"t={t}")
    blob = a.state_export()
    b = make_pool(capi, dict(meta, seed=999))
    b.state_import(blob)
    assert np.array_equal(b.state_export(), blob)
    for t in range(200):
        act = actions(rng, N)
        want = orc.step(act)
        eq(a.step(act), want, f"a t={t}")
        eq(b.step(act), want, f"b t={t}")


def test_large_pool_runs_the_128_thread_kernel(capi):
    """N = 300000 > 132 SMs * 8 * 128: the 128-thread step kernel.  The first and last 4096
    envs against the oracle (seeded seed + env id), and two env_id_offset halves must equal the
    full pool bit for bit."""
    import torch

    N, P, H, seed, T = 300000, 4096, 150000, 71, 40
    meta = meta_for("replay_cycle", N, seed)
    full = make_pool(capi, meta)
    lo = make_pool(capi, dict(meta, num_envs=H))
    hi = make_pool(capi, dict(meta, num_envs=H), env_id_offset=H)
    first = oracle_for(dict(meta, num_envs=P))
    from oracle.g2048_lib import Game2048Oracle

    last = Game2048Oracle(P, env_seed=np.arange(N - P, N) + seed,
                          max_episode_steps=meta["max_episode_steps"],
                          replay=cells(meta["replay_boards"], 512))
    rng = np.random.default_rng(17)
    for p in (full, lo, hi):
        p.reset_device()
    wf, wl = first.reset(), last.reset()
    for t in range(T + 1):
        torch.cuda.synchronize()
        got = outputs(full)
        glo, ghi = outputs(lo), outputs(hi)
        eq({k: v[:P] for k, v in got.items()}, wf, f"first t={t}")
        tail = {k: v[N - P:] for k, v in got.items()}
        wl_ids = dict(wl, **{"info:env_id": wl["info:env_id"] + N - P,
                             "info:players.env_id": wl["info:players.env_id"] + N - P})
        eq(tail, wl_ids, f"last t={t}")
        for k in got:
            assert np.array_equal(got[k][:H], glo[k]), (t, k)
            assert np.array_equal(got[k][H:], ghi[k]), (t, k)
        if t == T:
            break
        a = actions(rng, N)
        d = torch.from_numpy(a).cuda()
        full.step_device(d)
        lo.step_device(d[:H].contiguous())
        hi.step_device(d[H:].contiguous())
        wf, wl = first.step(a[:P]), last.step(a[N - P:])


def test_two_ranks_one_device(capi):
    import torch

    from envpool_b200._capi import _torch_view
    from envpool_b200.sharded import packed_views

    n, world = 1000, 2
    meta = meta_for("replay_cycle", world * n, 81)
    pools = [make_pool(capi, dict(meta, num_envs=n), env_id_offset=r * n) for r in range(world)]
    orc = oracle_for(meta)
    for r, p in enumerate(pools):
        p.exchange_init(world, r)
    bases = [p.exchange_base() for p in pools]
    for p in pools:
        p.exchange_attach(bases)
    rng = np.random.default_rng(19)
    want, acts = orc.reset(), None
    for t in range(60):
        d = None if acts is None else [torch.from_numpy(acts[r * n:(r + 1) * n].copy()).cuda()
                                       for r in range(world)]
        torch.cuda.synchronize()
        for r, p in enumerate(pools):
            p.step_exchange(None if d is None else d[r])
        ptrs = [p.exchange_wait() for p in pools]
        for p in pools:
            p.sync()
        for r, p in enumerate(pools):
            full = _torch_view(ptrs[r], (world, p.exchange_slice_bytes), torch.uint8, p.device)
            got = {k: v.reshape((world * n,) + tuple(v.shape[2:])).cpu().numpy()
                   for k, v in packed_views(full, p.keys, n).items()}
            eq(got, want, f"rank {r} t={t}")
        acts = actions(rng, world * n)
        want = orc.step(acts)
    for p in pools:
        steps, timed_out = p.exchange_status()
        assert steps == 60 and not timed_out


def test_boards_are_config_of_a_fresh_pool(capi):
    meta = meta_for("default", 8, 91)
    pool = make_pool(capi, meta)
    with pytest.raises(ValueError):
        pool.game2048_boards(np.full(16, 27, np.int32))
    pool.reset()
    with pytest.raises(capi.EpbError):
        pool.game2048_boards(np.zeros(16, np.int32))
    assert pool.bytes_per_env_step == 4 + 2 * (4 + 12) + 26 + 72 + 56


@pytest.mark.parametrize("action", [0, 1, 2, 3])
def test_reward_rounds_in_line_order(capi, action):
    """Line totals are added for lines 0..3: a 2^27 merge on line 0 swallows the three 2^2
    merges after it (half an ulp of 2^27 is 8); any other order keeps some of them.  The board
    is laid out so that line 0 of the direction holds the big merge."""
    base = np.zeros((4, 4), np.int32)
    base[0, :2] = 26
    base[1:, :2] = 1                         # rows: line i = row i when moving left
    board = {3: base, 1: base[:, ::-1], 0: base.T, 2: base.T[::-1, :]}[action]
    meta = dict(num_envs=1, seed=0, max_episode_steps=1000, add_random_cell=False,
                initial_board=",".join(map(str, board.ravel())), replay_boards="")
    pool, orc = make_pool(capi, meta), oracle_for(meta)
    eq(pool.reset(), orc.reset(), "reset")
    a = np.array([action], np.int32)
    want = orc.step(a)
    assert want["reward"][0] == np.float32(2.0**27)
    eq(pool.step(a), want, f"action {action}")


def test_lemire_rejection_in_the_random_cell(capi):
    """A crafted engine state: the random cell of one step reads words 100..103 of env 5's
    table, and word 102 is 0, which Lemire's method rejects for 14 empty cells, so word 103
    picks the cell.  The kernel must draw the same value and cell as the oracle and stand at
    word 104 after it."""
    from test_game2048 import crafted_state
    from test_oracle_rng_vs_libstdcxx import untemper

    N, e = 8, 5
    board = np.zeros(16, np.int32)
    board[[0, 1, 5]] = [1, 1, 3]             # moving left: 14 empty cells afterwards
    meta = dict(num_envs=N, seed=4, max_episode_steps=1000, add_random_cell=True,
                initial_board=",".join(map(str, board)), replay_boards="")
    pool, orc = make_pool(capi, meta), oracle_for(meta)
    eq(pool.reset(), orc.reset(), "reset")
    outs = [0x12345678, 0x01000000, 0, 0x9ABCDEF0]   # value 2 (canonical < 0.1), reject, pick
    blob = pool.state_export()
    st = pool.state_arrays(blob)
    assert st["mt_idx"][e] == 0                       # a configured reset draws nothing
    for k, o in enumerate(outs):
        st["mt"][(100 + k) // 8, e, (100 + k) % 8] = untemper(o)
    st["mt_idx"][e] = 100
    pool.state_import(blob)
    mt, idx = crafted_state(outs)
    orc.set_rng(e, mt, idx)
    a = np.full(N, 3, np.int32)
    want = orc.step(a)
    got = pool.step(a)
    eq(got, want, "step")
    after = got["obs:board"][e].ravel()
    assert after.max() == 3 and (after == 2).sum() == 2   # the merge (2) and a new tile 2
    assert pool.state_arrays(pool.state_export())["mt_idx"][e] == 104
