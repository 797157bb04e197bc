"""Record the PGX Chess / GardnerChess fixtures from the reference's own thread pool.

    python tests/golden/pgx/chess/make_chess_golden.py [CASE_PREFIX]   # needs oracle/_ref (build())

First scripts.json: pgx_chess_scripts.search's episode for each rule class of each game.  Then
per game, in the .npz format of ../go/make_go_golden.py (`meta`, `action` [T, n], every state key
as [T + 1, rows, ...], the legal-action mask bit-packed along its rows), except for obs: its 112
one-hot planes are bit-packed per player row (`obs_planes`) and its scalar channels (colour,
step_count / kMax, the castling rights, halfmove_count / 100) are stored once per player row
(`obs_scalars`), since they are constant across squares; `load` in tests/test_pgx_chess.py
rebuilds the float obs, and this recorder asserts that the rebuild is bit-exact.  obs is kept for
every `obs_every`-th record (`obs_steps`).  Cases:
  random    legal labels 70 % of the time, else any in-range label whose target lies on the board
            (25 %) or -1, the label count, INT_MIN, INT_MAX (5 %)
  legal     legal play: whole games, to the step limit where they last that long
  collide   legal play mixed with labels of the mover's own pieces that are not legal (onto its
            own pieces, blocked, into check) and with the illegal castle labels
  sequence  the scripts of tests/pgx_chess_scripts.py whose labels have their target on the
            board, one env each
Labels whose target lies off the board are never sent: the reference writes board[-1] for them.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path[:0] = [os.path.dirname(TESTS), TESTS]

from oracle import chess_lib  # noqa: E402

I32 = np.iinfo(np.int32)
PLANES = 112  # one-hot obs channels: 8 history steps x (12 piece planes + 2 repetition planes)


def cases(game):
    T = chess_lib.MAX_STEPS[game] + 2
    return {"random": dict(n=8, seed=3, T=120), "legal": dict(n=16, seed=5, T=T),
            "collide": dict(n=16, seed=11, T=100), "sequence": dict(seed=7)}


def on_board_labels(game):
    return np.flatnonzero(chess_lib.ChessOracle(game, 1, obs=False).on_board())


def legal_pick(rng, mask):
    return np.argmax(np.where(mask, rng.random(mask.shape), -1.0), axis=1).astype(np.int32)


def policy(game, case, rng, prev, t, on_board, script=None):
    mask = prev["info:legal_action_mask"]
    n, A = mask.shape
    if case == "sequence":
        return np.array([s[t] if t < len(s) else int(np.argmax(mask[i]))
                         for i, s in enumerate(script)], np.int32)
    a = legal_pick(rng, mask).astype(np.int64)
    u = rng.random(n)
    if case == "random":
        a = np.where(u < 0.3, on_board[rng.integers(0, len(on_board), n)], a)
        oor = np.array([-1, A, I32.min, I32.max])
        a = np.where(u < 0.05, oor[rng.integers(0, 4, n)], a)
    elif case == "collide":
        P, S = chess_lib.PLANES[game], chess_lib.SIZE[game]
        pos = np.arange(S * S)
        board = prev["info:board"][:, S - 1 - pos % S, pos // S]
        for e in range(n):
            own = np.flatnonzero(board[e] > 0)
            cand = [f * P + p for f in own for p in range(P)
                    if on_board_set[game][f * P + p] and not mask[e, f * P + p]]
            if u[e] < 0.25 and cand:
                a[e] = rng.choice(cand)
            elif u[e] < 0.28 and game == "Chess":
                a[e] = rng.choice([2364, 2367])
    return a.astype(np.int32)


on_board_set = {}


def pack_obs(game, obs):
    """[R, rows, S, S, C] float obs -> (bit-packed planes [R, rows, S S 112 / 8], scalars
    [R, rows, C - 112]); asserts the scalar channels are constant across squares and that
    unpack_obs gives the obs back bit for bit."""
    R, rows, S = obs.shape[0], obs.shape[1], obs.shape[2]
    planes = obs[..., :PLANES]
    assert np.isin(planes, (0.0, 1.0)).all()
    scalars = obs[..., PLANES:]
    assert (scalars == scalars[:, :, :1, :1]).all()
    packed = np.packbits(planes.astype(bool).reshape(R, rows, -1), axis=-1)
    sc = np.ascontiguousarray(scalars[:, :, 0, 0])
    assert np.array_equal(unpack_obs(packed, sc, S).view(np.uint32), obs.view(np.uint32))
    return packed, sc


def unpack_obs(packed, scalars, S):
    R, rows = packed.shape[:2]
    planes = np.unpackbits(packed, axis=-1, count=S * S * PLANES).reshape(R, rows, S, S, PLANES)
    sc = np.broadcast_to(scalars[:, :, None, None, :], (R, rows, S, S, scalars.shape[-1]))
    return np.concatenate([planes.astype(np.float32), sc.astype(np.float32)], axis=-1)


def record(game, case, cfg):
    import pgx_chess_scripts

    script = None
    if case == "sequence":
        on = chess_lib.ChessOracle(game, 1, obs=False)
        script = [s for s in pgx_chess_scripts.scripts(game).values()
                  if all(0 <= a < chess_lib.actions(game) and on.label_target(a) >= 0 or
                         not 0 <= a < chess_lib.actions(game) for a in s)]
    n = len(script) if script else cfg["n"]
    T = max(len(s) for s in script) + 3 if script else cfg["T"]
    rng = np.random.default_rng(cfg["seed"])
    on_board = on_board_labels(game)
    on_board_set[game] = np.zeros(chess_lib.actions(game), bool)
    on_board_set[game][on_board] = True
    ref = chess_lib.ChessRef(game, n, seed=cfg["seed"])
    outs = [ref.reset()]
    acts = []
    for t in range(T):
        a = policy(game, case, rng, outs[-1], t, on_board, script)
        acts.append(a)
        outs.append(ref.step(a))
    ref.close()
    data = {k: np.stack([o[k] for o in outs]) for k in outs[0]}
    every = 1 if T <= 130 else 8
    steps = np.arange(0, T + 1, every)
    obs = data.pop("obs")[steps]
    planes, scalars = pack_obs(game, obs)
    mask = data.pop("info:legal_action_mask")
    meta = {"game": game, "case": case, "num_envs": n, "seed": cfg["seed"], "steps": T,
            "obs_every": every, "obs_shape": list(obs.shape), "mask_shape": list(mask.shape)}
    path = os.path.join(HERE, f"{game}_{case}.npz")
    np.savez_compressed(path, meta=json.dumps(meta), action=np.stack(acts), obs_steps=steps,
                        obs_planes=planes, obs_scalars=scalars,
                        **{"info:legal_action_mask": np.packbits(mask.reshape(T + 1, n, -1), axis=-1)},
                        **data)
    return path


def main(only=None):
    """Every record, or those whose case name starts with `only` (command line argument)."""
    if not chess_lib.ref_available():
        sys.exit("oracle/_ref/libchess_ref.so is missing: run __graft_entry__.build() with an "
                 "envpool checkout")
    import pgx_chess_scripts

    if only is None:
        found = {g: pgx_chess_scripts.search(g) for g in chess_lib.GAMES}
        with open(pgx_chess_scripts.SCRIPTS_JSON, "w") as f:
            json.dump(found, f)
            f.write("\n")
    for game in chess_lib.GAMES:
        for case, cfg in cases(game).items():
            if only is None or case.startswith(only):
                print(record(game, case, cfg))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
