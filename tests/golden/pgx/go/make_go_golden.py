"""Record the PGX Go fixtures from the reference's own thread pool.

    python tests/golden/pgx/go/make_go_golden.py [CASE_PREFIX]   # needs oracle/_ref (build())

Per board size (oracle/go_lib.GAMES), in the .npz format of ../make_pgx_golden.py (`meta`,
`action` [T, n], every state key as [T + 1, rows, ...]) except that obs and the legal-action mask
are bit-packed along their flattened rows (`obs` / `info:legal_action_mask` hold np.packbits of
[T + 1, rows, -1]) and obs is kept for every `obs_every`-th record only (`obs_steps`).  Cases:
  random      legal actions 70 % of the time, else any of -1..S^2+1, INT_MIN and INT_MAX
  legal       legal play, passing 1 % of the time: full games up to 2 S^2 steps
  collide     legal play mixed with moves onto occupied cells, the ko point and suicides
  sequence    the scripts of tests/pgx_go_scripts.py, one env each
  komi_<k>    komi k in {0, -3.5, 0.5}: env 0 opens with two passes (equal areas S^2 : S^2), env 1
              with a black stone and two passes (black's area), env 2 with a pass, a white
              stone and two passes (white's area); then, and in every other env, the pass
              15 % of the time and a legal move otherwise, so double-pass ends are scored often
  mts_<m>     max_terminal_steps m in {1, 5, 2 S^2}: legal play
and psk_scripts.json: pgx_go_scripts.search_psk's superko episode per size.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path[:0] = [os.path.dirname(TESTS), TESTS]

from oracle import go_lib  # noqa: E402

I32 = np.iinfo(np.int32)
PSK_SEARCH = {"Go9x9": (256, 1), "Go13x13": (64, 2), "Go19x19": (32, 3)}  # (envs, seed)


def cases(game):
    S = go_lib.GAMES[game]
    A = S * S
    out = {"random": dict(n=8, seed=3, T=120), "legal": dict(n=4, seed=5, T=2 * A + 4),
           "collide": dict(n=16, seed=11, T=100), "sequence": dict(seed=7)}
    for k in (0.0, -3.5, 0.5):
        out[f"komi_{k:g}"] = dict(n=8, seed=13, T=80, komi=k)
    for m in (1, 5, 2 * A):
        out[f"mts_{m}"] = dict(n=4, seed=17, T=min(2 * m + 4, 2 * A + 4), max_terminal_steps=m)
    return out


def legal_pick(rng, mask, pass_p):
    A = mask.shape[1] - 1
    m = mask.copy()
    m[:, A] &= ~m[:, :A].any(1) | (rng.random(len(m)) < pass_p)
    return np.argmax(np.where(m, rng.random(m.shape), -1), axis=1).astype(np.int32)


def policy(case, rng, prev, t, script=None):
    mask = prev["info:legal_action_mask"]
    n, A = mask.shape[0], mask.shape[1] - 1
    if case.startswith("komi"):
        c = A // 2  # the centre cell
        a = np.where(rng.random(n) < 0.15, A, legal_pick(rng, mask, 0.0)).astype(np.int32)
        for e, opening in enumerate(([A, A], [c, A, A], [A, c, A, A])):
            if t < len(opening):
                a[e] = opening[t]
        return a
    if case == "sequence":
        return np.array([s[t] if t < len(s) else int(np.argmax(mask[i]))
                         for i, s in enumerate(script)], np.int32)
    if case == "random":
        a = legal_pick(rng, mask, 0.02).astype(np.int64)
        u = rng.random(n)
        a = np.where(u < 0.3, rng.integers(-1, A + 2, n), a)
        a = np.where(u < 0.02, np.where(rng.random(n) < 0.5, I32.min, I32.max), a)
        return a.astype(np.int32)
    if case == "collide":
        a = legal_pick(rng, mask, 0.01)
        board = prev["info:board"].reshape(n, -1)
        u = rng.random(n)
        for e in range(n):
            occ = np.flatnonzero(board[e])
            bad = np.flatnonzero((board[e] == 0) & ~mask[e, :A])
            if u[e] < 0.03 and occ.size:
                a[e] = rng.choice(occ)
            elif u[e] < 0.3 and prev["info:ko"][e] >= 0:
                a[e] = prev["info:ko"][e]
            elif u[e] < 0.06 and bad.size:
                a[e] = rng.choice(bad)
        return a
    return legal_pick(rng, mask, 0.01)


def record(game, case, cfg):
    from pgx_go_scripts import scripts

    script = list(scripts(game).values()) if case == "sequence" else None
    n = len(script) if script else cfg["n"]
    T = max(len(s) for s in script) + 3 if script else cfg["T"]
    kw = {k: cfg[k] for k in ("komi", "max_terminal_steps") if k in cfg}
    rng = np.random.default_rng(cfg["seed"])
    ref = go_lib.GoRef(game, n, seed=cfg["seed"], **kw)
    outs = [ref.reset()]
    acts = []
    for t in range(T):
        a = policy(case, rng, outs[-1], t, script)
        acts.append(a)
        outs.append(ref.step(a))
    ref.close()
    data = {k: np.stack([o[k] for o in outs]) for k in outs[0]}
    every = 1 if T <= 130 else 8
    steps = np.arange(0, T + 1, every)
    obs = data.pop("obs")[steps]
    mask = data.pop("info:legal_action_mask")
    meta = {"game": game, "case": case, "num_envs": n, "seed": cfg["seed"], "steps": T,
            "obs_every": every, "obs_shape": list(obs.shape), "mask_shape": list(mask.shape), **kw}
    path = os.path.join(HERE, f"{game}_{case}.npz")
    np.savez_compressed(path, meta=json.dumps(meta), action=np.stack(acts), obs_steps=steps,
                        obs=np.packbits(obs.reshape(len(steps), obs.shape[1], -1), axis=-1),
                        **{"info:legal_action_mask": np.packbits(mask.reshape(T + 1, n, -1), axis=-1)},
                        **data)
    return path


def main(only=None):
    """Every record, or those whose case name starts with `only` (command line argument)."""
    if not go_lib.ref_available():
        sys.exit("oracle/_ref/libgo_ref.so is missing: run __graft_entry__.build() with an envpool "
                 "checkout")
    from pgx_go_scripts import PSK_FILE, search_psk

    if only is None:
        psk = {g: search_psk(g, *PSK_SEARCH[g]) for g in go_lib.GAMES}
        with open(PSK_FILE, "w") as f:
            json.dump(psk, f)
            f.write("\n")
    for game in go_lib.GAMES:
        for case, cfg in cases(game).items():
            if only is None or case.startswith(only):
                print(record(game, case, cfg))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
