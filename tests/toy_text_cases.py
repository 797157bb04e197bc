"""Crafted toy_text pools: every reachable (state, action) pair of each env, paired with an
mt19937 table whose next outputs sit on the env's draw boundaries.  Shared by the CPU
coverage test (test_toy_text_crafted.py) and the engine comparison (test_gpu_toy_text.py).

Crafting a table: words 0..K zero and words 397..397+K-1 the untempered wanted outputs make
the next regeneration (engine: mt_idx = 0, chunk by chunk; std::mt19937: position 624, the
whole table) emit exactly those K outputs, for any K <= 200.  New word i is
    old[i + 397] ^ twist(old[i] & 0x80000000 | old[i + 1] & 0x7fffffff),
and twist(0) = 0; old[i + 397] has not been regenerated yet while i + 397 < 624, and chunk
i // 8 of the engine reads the same three old words.  Every later word regenerates the same
way on both sides because the whole 624-word table is the same.

A case packs each state twice: into the engine's words (istate, flags = cur << 1 | done,
written through state_arrays / state_import) and into the oracle's fields (set_int_states)."""
import functools
import itertools
import zlib

import numpy as np

MAX_FORCED = 200
MAX_POOL = 65536   # rows per pool: bounds the oracle's memory (one 2.5 KB table per env)
STEPS = 10         # FrozenLake: step 1 fills the slip queue, steps 2-8 pop it, step 9 refills
F = 0xFFFFFFFF


def untemper(y):
    """Inverse of mt19937's output tempering, elementwise over a uint32 array."""
    y = np.asarray(y, dtype=np.uint64) & F
    y = y ^ (y >> 18)
    y = y ^ ((y << 15) & 0xEFC60000)
    t = y
    for _ in range(5):
        t = y ^ ((t << 7) & 0x9D2C5680)
    y = t & F
    t = y
    for _ in range(3):
        t = y ^ (t >> 11)
    return (t & F).astype(np.uint32)


def crafted_tables(rng, outputs, distinct=64):
    """[N, 624] tables whose next len(outputs[e]) outputs are outputs[e] (K <= 200 each).
    The words nothing forces come from `distinct` random tables, reused round robin."""
    outputs = np.asarray(outputs, dtype=np.uint64)
    n, k = outputs.shape
    assert k <= MAX_FORCED
    base = rng.integers(0, 2**32, size=(min(n, distinct), 624), dtype=np.uint32)
    mt = base[np.arange(n) % base.shape[0]]
    mt[:, 0:k + 1] = 0
    mt[:, 397:397 + k] = untemper(outputs)
    return mt


def crafted_table(rng, outputs):
    """One table whose next len(outputs) outputs are `outputs`."""
    return crafted_tables(rng, [list(outputs)], distinct=1)[0]


def load_engine(pool, tables, istate=None, flags=None, force_done=False):
    """Engine side of a crafted pool: tables [N, 624] go into the chunked [78][N][8] layout with
    mt_idx = 0; istate [NI, N] and flags [N] replace the env state when given.  Returns the
    imported blob."""
    blob = pool.state_export()
    st = pool.state_arrays(blob)
    n = tables.shape[0]
    st["mt"][:] = tables.reshape(n, 78, 8).transpose(1, 0, 2)
    st["mt_idx"][:] = 0
    if "rprod" in st:
        # classic_control keeps each env's NEXT initial states in a ring of records drawn from
        # the table before the crafting; emptying the ring makes epb_state_import redraw all
        # of them from the crafted table (the refill path), as the oracle's next Resets will
        st["rprod"][:] = st["rcons"]
    if istate is not None:
        st["istate"][:] = istate
    if flags is not None:
        st["flags"][:] = flags
    if force_done:
        st["flags"][:] = st["flags"] | 1
    pool.state_import(blob)
    return blob


def load_oracle(orc, tables, state=None, force_done=False):
    """Oracle side: every env's std::mt19937 at position 624 of its crafted table; `state` (the
    dict OraclePool.set_int_states takes) replaces the toy_text state when given."""
    if state is not None:
        orc.set_int_states(state)
    for e in range(tables.shape[0]):
        orc.set_rng(e, tables[e], 624)
        if force_done:
            s5, _, cur = orc.get_state(e)
            orc.set_state(e, s5, 1, cur)


def load_both(pool, orc, tables, force_done=False, case=None):
    """The same crafted tables (and, given a Case, the same states) into engine and oracle."""
    if case is None:
        load_engine(pool, tables, force_done=force_done)
        load_oracle(orc, tables, force_done=force_done)
    else:
        load_engine(pool, tables, case.istate, case.flags, force_done)
        load_oracle(orc, tables, case.ostate, force_done)


# ------------------------------------------------------------------------ boundary words
def lemire_boundaries(r):
    """For uniform_int over a range of r values: the first word of every result and the word
    just below it (result = (w * r) >> 32), plus the two extreme accepted words."""
    out = {1, F}
    for k in range(1, r):
        w = -(-(k << 32) // r)
        out.update((w - 1, w))
    return sorted(out)


def lemire_rejected(r):
    """The words uniform_int(0, r - 1) rejects: (w * r) mod 2^32 < 2^32 mod r."""
    thr = (1 << 32) % r
    inv = pow(r, -1, 1 << 32)
    return [(k * inv) % (1 << 32) for k in range(thr)]


# range 3 (FrozenLake's and slippery CliffWalking's slip): 0 is the only rejected word
SLIP_WORDS = [1, 0x55555555, 0x55555556, 0xAAAAAAAA, 0xAAAAAAAB, F]
SLIP_OFFSET = {1: -1, 0x55555555: -1, 0x55555556: 0, 0xAAAAAAAA: 0, 0xAAAAAAAB: 1, F: 1}
# first forced words of a slip row: each boundary word, then the rejected 0 once and twice in a
# row in front of a boundary word (None: drawn from SLIP_WORDS)
SLIP_HEADS = [(w,) for w in SLIP_WORDS] + [(0, None), (0, 0, None)]
# NChain: (d1, d2) pairs and whether canonical(d1, d2) < 0.2, i.e. the action slips
NCHAIN_PAIRS = [
    ((0x33333400, 0x33333333), False),   # exactly 0.2
    ((0x33333200, 0x33333333), True),    # one ulp below 0.2
    ((0x33333300, 0x33333333), False),   # midpoint: round half to even gives 0.2
    ((0, 0), True),                      # 0.0
    ((F, F), False),                     # >= 1: clamped to nextafter(1, 0)
]
BLACKJACK_WORDS = lemire_boundaries(13) + lemire_rejected(13)
CATCH_WORDS = lemire_boundaries(5) + lemire_rejected(5)
TAXI_WORDS = sorted(set(lemire_boundaries(5) + lemire_boundaries(4) + lemire_rejected(5)))


class Case:
    """One crafted pool: rows are (state, first action) pairs.  istate [NI, N] / flags [N] are
    the engine's words, ostate the oracle's fields, act0 [N] the first step's actions, heads
    the forced-word pattern of each row, tables [N, 624]."""

    def __init__(self, name, task, iopt, max_episode_steps, n_act):
        self.name, self.task, self.iopt, self.ms, self.n_act = (name, task, iopt,
                                                                max_episode_steps, n_act)

    @property
    def n(self):
        return len(self.flags)

    def kwargs(self):
        return dict(max_episode_steps=self.ms, iopt=self.iopt)

    def actions(self):
        """[STEPS, N]: act0, then seeded random actions."""
        rng = np.random.default_rng(zlib.crc32(self.name.encode()))
        a = rng.integers(0, self.n_act, size=(STEPS, self.n)).astype(np.int32)
        a[0] = self.act0
        return a


def _plain(case, rows, fields, heads, fill, k, seed, pack):
    """Fills a one-word-state Case.  rows: (state tuple, first action, head index, cur, done);
    the state tuple's first `fields` entries are the oracle's i[0..]; pack(state) gives the
    engine's words.  Forced words: K drawn from `fill` (a word list, or fill(rng, n, K)), then
    each row's head pattern over the first ones."""
    n = len(rows)
    case.act0 = np.array([r[1] for r in rows], np.int32)
    case.heads = np.array([r[2] for r in rows], np.int32)
    cur = np.array([r[3] for r in rows], np.int32)
    done = np.array([r[4] for r in rows], np.int32)
    case.flags = (cur << 1) | done
    case.istate = np.stack([pack(r[0]) for r in rows], axis=1).astype(np.int32)
    case.ostate = {"i": np.zeros((n, 8), np.int32), "done": done, "cur": cur}
    for j in range(fields):
        case.ostate["i"][:, j] = [r[0][j] for r in rows]
    rng = np.random.default_rng(seed)
    if callable(fill):
        words = fill(rng, n, k)
    else:
        words = rng.choice(np.array(fill, dtype=np.uint64), size=(n, k))
    for h, head in enumerate(heads):
        sel = case.heads == h
        for j, w in enumerate(head):
            if w is not None:
                words[sel, j] = w
    case.forced = words
    case.tables = crafted_tables(rng, words)
    return case


LAKE4 = ["SFFF", "FHFH", "FFFH", "HFFG"]
LAKE8 = ["SFFFFFFF", "FFFFFFFF", "FFFHFFFF", "FFFFFHFF",
         "FFFHFFFF", "FHHFFFHF", "FHFFHFHF", "FFFHFFFG"]


def frozen_lake(size):
    lake = LAKE4 if size == 4 else LAKE8
    cells = [(x, y) for x in range(size) for y in range(size) if lake[x][y] in "SF"]
    rows = [(c, a, h, cur, 0) for c, a, h, cur in
            itertools.product(cells, range(4), range(len(SLIP_HEADS)), (0, 50, 98, 99))]
    case = Case(f"FrozenLake{size}", "FrozenLake", size, 100, 4)
    # empty slip queue (marker bit only): the first step draws 8 words from the crafted table
    return _plain(case, rows, 2, SLIP_HEADS, SLIP_WORDS + [0], 24, size,
                  lambda s: [s[0] | s[1] << 3 | 1 << 6])


def catch():
    states = list(itertools.product(range(9), range(5), range(5)))
    rows = [(s, a, 0, s[0], done) for done, s, a in itertools.product((0, 1), states, range(3))]
    case = Case("Catch", "Catch", -1, -1, 3)
    return _plain(case, rows, 3, [()], CATCH_WORDS, 16, 6,
                  lambda s: [s[0] | s[1] << 8 | s[2] << 16])


def taxi():
    states = list(itertools.product(range(5), range(5), range(5), range(4)))
    rows = [(s, a, 0, cur, 0) for s, a, cur in itertools.product(states, range(6), (0, 198, 199))]
    case = Case("Taxi", "Taxi", -1, 200, 6)
    return _plain(case, rows, 4, [()], TAXI_WORDS, 16, 7,
                  lambda s: [s[0] | s[1] << 4 | s[2] << 8 | s[3] << 12])


def nchain():
    heads = [p for p, _ in NCHAIN_PAIRS]
    rows = [((s,), a, h, cur, 0) for s, a, h, cur, _ in
            itertools.product(range(5), range(2), range(len(heads)), (0, 998, 999), range(4))]
    case = Case("NChain", "NChain", -1, 1000, 2)
    def fill(rng, n, k):  # later draws: whole crafted pairs
        pick = rng.integers(0, len(heads), size=(n, k // 2))
        return np.array(heads, dtype=np.uint64)[pick].reshape(n, k)

    return _plain(case, rows, 1, heads, fill, 24, 8, lambda s: [s[0]])


def cliff_walking(slippery):
    cells = [(x, y) for x in range(3) for y in range(12)] + [(3, 0)]
    heads = SLIP_HEADS if slippery else [()]
    rows = [(c, a, h, cur, 0) for c, a, h, cur in
            itertools.product(cells, range(4), range(len(heads)), (0, 7))]
    case = Case("CliffWalkingSlippery" if slippery else "CliffWalking", "CliffWalking",
                int(slippery), -1, 4)
    return _plain(case, rows, 2, heads, SLIP_WORDS + [0], 24, 9 + slippery,
                  lambda s: [s[0] | s[1] << 8])


# ---------------------------------------------------------------------------- Blackjack
def _sum_hand(raw, ace):
    return raw + 10 if ace and raw + 10 <= 21 else raw


@functools.lru_cache(maxsize=None)
def player_hands():
    """Every reachable player hand class (raw sum, has-ace, card count, first two cards) with
    one card list that realises it: two cards, then hits while the hand is not bust."""
    seen, todo = {}, []
    for c0, c1 in itertools.product(range(1, 11), repeat=2):
        key = (c0 + c1, int(c0 == 1 or c1 == 1), 2, c0, c1)
        if key not in seen:
            seen[key] = [c0, c1]
            todo.append(key)
    while todo:
        key = todo.pop()
        raw, ace, n, c0, c1 = key
        for c in range(1, 11):
            nk = (raw + c, ace | (c == 1), n + 1, c0, c1)
            if nk not in seen and _sum_hand(nk[0], nk[1]) <= 21:
                seen[nk] = seen[key] + [c]
                todo.append(nk)
    return tuple(seen[k] for k in sorted(seen))


def _pack_hand(cards):
    """Engine hand word: sum | ace << 6 | n << 7 | c0 << 12 | c1 << 16."""
    return (sum(cards) | int(1 in cards) << 6 | len(cards) << 7 | cards[0] << 12 |
            cards[1] << 16)


# one dealer pair per up-card, and player hands beside every dealer pair: naturals both ways,
# soft and hard totals, 21 of three cards, a long all-ace hand
UPCARD_PAIRS = [(c, 10 if c != 10 else 7) for c in range(1, 11)]
PLAYER_PICKS = [[1, 10], [10, 1], [10, 10], [9, 7], [2, 3], [1, 5], [10, 6, 5], [1, 1],
                [5, 5, 1], [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1]]


def blackjack(option):
    """All pools of one (natural, sab) option: option = natural | sab << 1."""
    rows = list(itertools.product(player_hands(), UPCARD_PAIRS, range(2)))
    rows += itertools.product(PLAYER_PICKS, itertools.product(range(1, 11), repeat=2), range(2))
    cases = []
    for part, lo in enumerate(range(0, len(rows), MAX_POOL)):
        chunk = rows[lo:lo + MAX_POOL]
        n = len(chunk)
        case = Case(f"Blackjack{option}.{part}", "Blackjack", option, -1, 2)
        case.act0 = np.array([r[2] for r in chunk], np.int32)
        case.heads = np.zeros(n, np.int32)
        cur = np.full(n, 1, np.int32)
        case.flags = cur << 1
        case.istate = np.array([[_pack_hand(p) for p, _, _ in chunk],
                                [_pack_hand(list(d)) for _, d, _ in chunk]], np.int32)
        st = {"i": np.zeros((n, 8), np.int32), "done": np.zeros(n, np.int32), "cur": cur,
              "player": np.zeros((n, 32), np.int32), "dealer": np.zeros((n, 32), np.int32),
              "nplayer": np.array([len(p) for p, _, _ in chunk], np.int32),
              "ndealer": np.full(n, 2, np.int32)}
        for j, (p, d, _) in enumerate(chunk):
            st["player"][j, :len(p)] = p
            st["dealer"][j, :2] = d
        case.ostate = st
        rng = np.random.default_rng(100 + 10 * option + part)
        case.forced = rng.choice(np.array(BLACKJACK_WORDS, dtype=np.uint64), size=(n, 24))
        case.tables = crafted_tables(rng, case.forced)
        cases.append(case)
    return cases


def builders():
    """name -> zero-argument function returning the list of Cases of that env variant."""
    out = {"FrozenLake4": lambda: [frozen_lake(4)], "FrozenLake8": lambda: [frozen_lake(8)],
           "Catch": lambda: [catch()], "Taxi": lambda: [taxi()], "NChain": lambda: [nchain()],
           "CliffWalking": lambda: [cliff_walking(False)],
           "CliffWalkingSlippery": lambda: [cliff_walking(True)]}
    for opt in range(4):
        out[f"Blackjack{opt}"] = lambda opt=opt: blackjack(opt)
    return out


VARIANTS = sorted(builders())


def oracle_run(case, every_state=True):
    """The oracle on a crafted case: (outputs of every step, oracle integer states after every
    step -- or, every_state False, after the last step only)."""
    from oracle.oracle_lib import OraclePool

    orc = OraclePool(case.task, case.n, seed=0, **case.kwargs())
    load_oracle(orc, case.tables, case.ostate)
    outs, states = [], []
    for t, a in enumerate(case.actions()):
        outs.append(orc.step(a))
        if every_state or t == STEPS - 1:
            states.append(orc.int_states())
    orc.close()
    return outs, states
