"""GPU: Jumanji Minesweeper-v0 on the sm_90a kernel (envpool_b200/csrc/jumanji.cu), bit for bit
against the oracle (oracle/ms_oracle.c), the reference's own thread pool (oracle/_ref, when the
build made it) and the fixtures recorded from it, through every entry point of the engine."""
import numpy as np
import pytest

from helpers import assert_batch_equal
from test_minesweeper import FIXTURES, load_fixture, oracle_for, parse_config

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
REPLAY = ",".join(str(v) for v in np.random.default_rng(7).integers(-1, 9, size=500))
CONFIGS = {
    "default": dict(max_episode_steps=90, mine_locations="", replay_boards="",
                    replay_rewards="", replay_done=""),
    "configured": dict(max_episode_steps=90, mine_locations="5,5,17,-3,100,33,0,99,44,45,54",
                       replay_boards="", replay_rewards="", replay_done=""),
    # 5 replay boards, the third one ends the episode; max_episode_steps 3 truncates it
    "replay": dict(max_episode_steps=3, mine_locations="", replay_boards=REPLAY,
                   replay_rewards="0.5,-2.25,7", replay_done="0,False,true"),
    # all 32 replay steps (boards 5..31 unexplored), then the env plays on
    "replay_long": dict(max_episode_steps=90, mine_locations="", replay_boards=REPLAY,
                        replay_rewards="1", replay_done=""),
}


def meta_for(config, n, seed):
    return dict(CONFIGS[config], num_envs=n, seed=seed)


def make_pool(capi, meta, **kw):
    pool = capi.CPool("Minesweeper", meta["num_envs"], seed=meta["seed"],
                      max_episode_steps=meta["max_episode_steps"], **kw)
    mines, replay, rewards, done = parse_config(meta)
    if mines is not None or replay is not None:
        pool.minesweeper_config(mines, replay, rewards, done)
    return pool


def ref_for(meta):
    """The reference's own AsyncEnvPool<MinesweeperEnv> when the build compiled it, else None."""
    from oracle import ms_lib

    if not ms_lib.ref_available():
        return None
    return ms_lib.MinesweeperRef(meta["num_envs"], seed=meta["seed"],
                                 max_episode_steps=meta["max_episode_steps"],
                                 mine_locations=meta["mine_locations"],
                                 replay_boards=meta["replay_boards"],
                                 replay_rewards=meta["replay_rewards"],
                                 replay_done=meta["replay_done"], num_threads=4)


def actions(rng, shape):
    """(row, column) uniform in [0, 9], one component in ten out of range (the env clamps)."""
    a = rng.integers(0, 10, size=tuple(np.atleast_1d(shape)) + (2,)).astype(np.int64)
    odd = rng.random(a.shape) < 0.1
    a[odd] = rng.choice(np.array([-5, 10, INT32_MIN, INT32_MAX]), size=int(odd.sum()))
    return a.astype(np.int32)


def outputs(pool, n=None):
    return {k: v.cpu().numpy() for k, v in pool.outputs_torch(n).items()}


def eq(got, want, ctx):
    assert_batch_equal(got, want, "Minesweeper", 0.0, ctx)


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_random_rollouts_match_oracle_and_reference(capi, config):
    meta = meta_for(config, 2048, 21)
    pool, orc, ref = make_pool(capi, meta), oracle_for(meta), ref_for(meta)
    rng = np.random.default_rng(5)
    want = orc.reset()
    eq(pool.reset(), want, f"{config} reset")
    if ref is not None:
        eq(ref.reset(), want, f"{config} reference reset")
    for t in range(300):
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


def _kwargs(meta):
    return dict(num_envs=meta["num_envs"], seed=meta["seed"],
                max_episode_steps=meta["max_episode_steps"],
                minesweeper_mine_locations=meta["mine_locations"],
                minesweeper_replay_boards=meta["replay_boards"],
                minesweeper_replay_rewards=meta["replay_rewards"],
                minesweeper_replay_done=meta["replay_done"])


@pytest.mark.parametrize("name", ["default", "short_replay", "max_steps_5"])
def test_reference_fixtures_through_make_gymnasium_and_make_dm(capi, name):
    import envpool_b200 as ep

    meta, gold = load_fixture(name)
    obs_keys = ["board", "action_mask", "num_mines", "step_count"]
    env = ep.make_gymnasium("Minesweeper-v0", **_kwargs(meta))
    assert set(env.observation_space.keys()) == set(obs_keys)
    obs, info = env.reset()
    for k in obs_keys:
        np.testing.assert_array_equal(obs[k], gold["obs:" + k][0], k)
    for t, a in enumerate(gold["actions"]):
        obs, rew, term, trunc, info = env.step(a)
        for k in obs_keys:
            np.testing.assert_array_equal(obs[k], gold["obs:" + k][t + 1], f"{k} t={t}")
        np.testing.assert_array_equal(rew, gold["reward"][t + 1])
        np.testing.assert_array_equal(term | trunc, gold["done"][t + 1])
        np.testing.assert_array_equal(trunc, gold["trunc"][t + 1])
        np.testing.assert_array_equal(info["elapsed_step"], gold["elapsed_step"][t + 1])
    dm = ep.make_dm("Minesweeper-v0", **_kwargs(meta))
    ts = dm.reset()
    assert list(ts.observation._fields) == ["env_id", "players"] + obs_keys
    for t, a in enumerate(gold["actions"]):
        ts = dm.step(a)
        for k in obs_keys:
            np.testing.assert_array_equal(getattr(ts.observation, k), gold["obs:" + k][t + 1])
        np.testing.assert_array_equal(ts.reward, gold["reward"][t + 1])
        np.testing.assert_array_equal(ts.step_type, gold["step_type"][t + 1])


@pytest.mark.parametrize("config", ["default", "replay"])
def test_every_entry_point_is_bit_identical(capi, config):
    """One action stream [T, N, 2] through host step, step_device, step_many_device (graph and
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


def test_odd_pool_rollout_and_unaligned_action_rows(capi):
    """N = 1001: rollout rows of the 100-byte mask column start at 4-byte (not 16-byte)
    offsets; and a device action buffer that starts 4 bytes past an 8-byte boundary."""
    import torch

    N, T = 1001, 30
    meta = meta_for("configured", N, 33)
    rng = np.random.default_rng(9)
    acts = actions(rng, (T, N))
    orc = oracle_for(meta)
    orc.reset()
    want = [orc.step(acts[t]) for t in range(T)]
    roll = make_pool(capi, meta)
    roll.reset_device()
    tdt = {np.dtype(np.int32): torch.int32, np.dtype(np.float32): torch.float32,
           np.dtype(np.bool_): torch.bool}
    cols = [torch.empty((T, N) + k.shape, dtype=tdt[k.dtype], device="cuda") for k in roll.keys]
    roll.rollout_device(torch.from_numpy(acts).cuda(), T, cols)
    roll.sync()
    for t in range(T):
        eq({k.name: c[t].cpu().numpy() for k, c in zip(roll.keys, cols)}, want[t], f"t={t}")
    dev = make_pool(capi, meta)
    dev.reset_device()
    flat = torch.zeros(2 * N + 1, dtype=torch.int32, device="cuda")
    for t in range(T):
        flat[1:].copy_(torch.from_numpy(acts[t].ravel()).cuda())
        dev.step_device(flat.data_ptr() + 4)
        torch.cuda.synchronize()
        eq(outputs(dev), want[t], f"unaligned t={t}")


def test_async_send_recv_with_smaller_batches(capi):
    N, B = 1024, 256
    meta = meta_for("replay", N, 41)
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


@pytest.mark.parametrize("config", ["default", "replay"])
def test_snapshot_continues_in_a_pool_with_another_seed(capi, config):
    """The blob carries the configuration too: the second pool is built without it."""
    N = 1500
    meta = meta_for(config, N, 61)
    a, orc = make_pool(capi, meta), oracle_for(meta)
    rng = np.random.default_rng(13)
    eq(a.reset(), orc.reset(), "reset")
    for t in range(57):
        act = actions(rng, N)
        eq(a.step(act), orc.step(act), f"t={t}")
    blob = a.state_export()
    # max_episode_steps is a pool option, not state: the second pool is built with the same
    b = make_pool(capi, dict(meta_for("default", N, 999),
                             max_episode_steps=meta["max_episode_steps"]))
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

    from oracle.ms_lib import MinesweeperOracle

    N, P, H, seed, T = 300000, 4096, 150000, 71, 40
    meta = meta_for("default", N, seed)
    full = make_pool(capi, meta)
    lo = make_pool(capi, dict(meta, num_envs=H))
    hi = make_pool(capi, dict(meta, num_envs=H), env_id_offset=H)
    first = oracle_for(dict(meta, num_envs=P))
    last = MinesweeperOracle(P, env_seed=np.arange(N - P, N) + seed,
                             max_episode_steps=meta["max_episode_steps"])
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
    meta = meta_for("replay", world * n, 81)
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


def test_config_of_a_fresh_pool_and_bytes_per_step(capi):
    meta = meta_for("default", 8, 91)
    pool = make_pool(capi, meta)
    with pytest.raises(ValueError):
        pool.minesweeper_config(replay_boards=np.full(3200, 9, np.int32))
    with pytest.raises(ValueError):
        pool.minesweeper_config(replay_boards=np.full(3200, -2, np.int32))
    pool.reset()
    with pytest.raises(capi.EpbError):
        pool.minesweeper_config(mines=np.ones(100, np.int32))
    assert pool.bytes_per_env_step == 8 + 2 * (4 + 68) + 26 + 508
    assert pool.action_key.row_bytes == 8 and pool.action_key.shape == (2,)


def test_hand_built_boards_on_the_kernel(capi):
    """The oracle's Reveal cases on the kernel: a wall of mines (corner flood stops at the
    numbers), one mine (a full flood solves the board), a mine click; then a board loaded
    through the state blob (packed as jumanji.cu documents) with an explored wall the flood
    must not cross."""
    cases = {
        "wall": (list(range(3, 100, 10)), [(0, 0), (5, 2)]),
        "one mine": ([55], [(9, 0)]),
        "mine click": ([0, 1, 10], [(0, 0), (0, 0), (1, 1)]),
    }
    for name, (cells, clicks) in cases.items():
        meta = dict(CONFIGS["default"], num_envs=1, seed=0,
                    mine_locations=",".join(map(str, cells)))
        pool, orc = make_pool(capi, meta), oracle_for(meta)
        eq(pool.reset(), orc.reset(), f"{name} reset")
        for r, c in clicks:
            a = np.array([[r, c]], np.int32)
            eq(pool.step(a), orc.step(a), f"{name} click {(r, c)}")

    meta = dict(CONFIGS["default"], num_envs=4, seed=0, mine_locations="99")
    pool, orc = make_pool(capi, meta), oracle_for(meta)
    eq(pool.reset(), orc.reset(), "reset")
    board = np.full(100, -1, np.int32)
    board[4::10] = 0
    blob = pool.state_export()
    ist = pool.state_arrays(blob)["istate"]
    words = np.zeros(13, np.uint32)
    for c in range(100):
        words[c // 8] |= np.uint32((board[c] + 1) << (4 * (c % 8)))
    for e in range(4):
        ist[:13, e] = words.view(np.int32)
        orc.set_board(e, board)
    pool.state_import(blob)
    a = np.array([[0, 0], [0, 9], [9, 9], [5, 4]], np.int32)
    want = orc.step(a)
    eq(pool.step(a), want, "set board")
    assert (want["obs:board"][0][:, :4] == 0).all() and (want["obs:board"][0][:, 5:] == -1).all()
