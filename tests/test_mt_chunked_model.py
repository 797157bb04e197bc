"""CPU: the lazy, chunk-wise regeneration of the mt19937 table that the device RNG uses
(envpool_b200/csrc/common.cuh, `struct Mt`; DESIGN.md section 1) produces std::mt19937's
sequence.  The scheme is restated here in numpy, 8-word chunks and all, and run for three
full table cycles against the oracle's block-twist generator (itself pinned to libstdc++
through the reference build and the C++ standard's 10000th-draw known answer).

Device layout: chunk c of an env = the 8 words 8c..8c+7.  A chunk is regenerated when the
read position enters it, from values it finds in the table at that moment:
  word i needs  old[i], old[i+1]  and  table[(i+397) % 624]
  * i+1 inside the chunk: its OLD value (the whole chunk is computed from loaded old words);
  * i+1 = first word of the next chunk: not regenerated yet (old) -- except after word 623,
    whose successor is word 0 of the NEW block, exactly what the block twist uses;
  * i+397 < 624: a later chunk, still old;  i+397 >= 624: an earlier chunk, already new --
    again what the block twist uses.
"""
import numpy as np

N, M = 624, 397
UPPER, LOWER, MAG = np.uint32(0x80000000), np.uint32(0x7FFFFFFF), np.uint32(0x9908B0DF)


def init_genrand(seed):
    mt = np.zeros(N, dtype=np.uint32)
    s = np.uint64(seed & 0xFFFFFFFF)
    mt[0] = s
    for i in range(1, N):
        s = (np.uint64(1812433253) * (s ^ (s >> np.uint64(30))) + np.uint64(i)) \
            & np.uint64(0xFFFFFFFF)
        mt[i] = s
    return mt


def temper(y):
    y = np.uint32(y)
    y ^= y >> np.uint32(11)
    y ^= (y << np.uint32(7)) & np.uint32(0x9D2C5680)
    y ^= (y << np.uint32(15)) & np.uint32(0xEFC60000)
    y ^= y >> np.uint32(18)
    return int(y)


class ChunkedMt:
    """table[78][8] + read position, regenerated one chunk at a time (device scheme)."""

    def __init__(self, seed):
        self.table = init_genrand(seed).reshape(N // 8, 8)
        self.idx = 0          # seed_kernel: "the first draw regenerates word 0"
        self.loads = 0

    def enter_chunk(self, c):
        flat = self.table.reshape(-1)
        base = 8 * c
        own = flat[base:base + 8].copy()                 # sector 1: own chunk (old)
        nxt = flat[(base + 8) % N]                       # sector 2: first word of the next
        far = np.array([flat[(base + k + M) % N] for k in range(8)], dtype=np.uint32)
        self.loads += 4                                  # sectors 3,4: the i+397 window
        new = np.empty(8, dtype=np.uint32)
        for k in range(8):
            succ = own[k + 1] if k < 7 else nxt
            y = (own[k] & UPPER) | (succ & LOWER)
            new[k] = far[k] ^ (y >> np.uint32(1)) ^ (MAG if (y & np.uint32(1)) else np.uint32(0))
        flat[base:base + 8] = new                        # one sector write

    def next(self):
        if self.idx % 8 == 0:
            self.enter_chunk((self.idx % N) // 8)
        v = self.table.reshape(-1)[self.idx % N]
        self.idx = (self.idx + 1) % N if self.idx + 1 != N else 0
        return temper(v)


def test_chunked_regeneration_equals_std_mt19937():
    from oracle.oracle_lib import OraclePool

    for seed in (0, 7, 5489, 2**31 - 1):
        orc = OraclePool("CartPole", 1, seed=seed, max_episode_steps=500)
        dev = ChunkedMt(seed)
        got = [dev.next() for _ in range(3 * N + 17)]
        want = [orc.draw(0) for _ in range(3 * N + 17)]
        assert got == want, (seed, next(i for i, (a, b) in enumerate(zip(got, want)) if a != b))
        assert dev.loads == 4 * ((3 * N + 17 + 7) // 8)   # 4 sector reads per 8 draws


def test_window_never_straddles_regenerated_and_old_words_wrongly():
    """The 8-word i+397 window of a chunk lies in at most two chunks, and for every word the
    table holds the value the block twist would use at that moment (old if i+397 < 624, new
    otherwise) -- checked structurally: within one chunk regeneration no needed word has
    been overwritten earlier in the same chunk."""
    for c in range(N // 8):
        need = {(8 * c + k + M) % N for k in range(8)} | {(8 * c + 8) % N}
        own = set(range(8 * c, 8 * c + 8))
        assert not (need & own), c
        assert len({w // 8 for w in need if w != (8 * c + 8) % N}) <= 2, c


def test_slip_queue_equals_sequential_lemire_including_rejections():
    """FrozenLake draws one uniform_int(-1, 1) per step.  libstdc++'s Lemire loop
    (uniform_int_dist.h:252-282, range 3 on a 32-bit engine) rejects exactly the word 0 and
    redraws; the device kernel (csrc/toytext.cu FrozenLake::pop_slip) turns 8 engine words at
    a time into 2-bit codes under a marker bit ("3" = rejected word) and pops one code per
    step.  A rejection has probability 2^-32 per draw, so no sampled GPU test ever reaches it:
    here both algorithms run on word streams with zeros injected (also at chunk boundaries and
    back to back) and must produce the same results from the same number of consumed words."""
    rng = np.random.default_rng(0)

    def sequential(words):
        out, i = [], 0
        while True:
            while i < len(words):
                w = int(words[i])
                i += 1
                p = w * 3
                lo = p & 0xFFFFFFFF
                if lo < 3 and lo < ((1 << 32) - 3) % 3:      # t = (2^32 - r) % r = 1
                    continue                                   # redraw
                out.append((p >> 32) - 1)
                break
            else:
                return out

    def queued(words):
        out, i, queue = [], 0, 1                                # marker bit only = empty
        while True:
            if queue <= 1:
                if i + 8 > len(words):
                    return out
                chunk = words[i:i + 8]
                i += 8
                queue = 1
                for k in range(7, -1, -1):
                    w = int(chunk[k])
                    code = 3 if w == 0 else (w * 3) >> 32
                    queue = (queue << 2) | code
                assert queue < (1 << 17)                        # fits beside x|y<<3 in an int32
            code = queue & 3
            queue >>= 2
            if code != 3:
                out.append(code - 1)

    for trial in range(50):
        words = rng.integers(0, 2**32, size=8 * 40, dtype=np.uint64)
        zeros = rng.choice(len(words), size=rng.integers(0, 40), replace=False)
        words[zeros] = 0
        if trial % 5 == 0:
            words[8:19] = 0                                     # a whole chunk and a half
        a, b = sequential(words), queued(words)
        assert b == a[:len(b)] and len(a) - len(b) <= 8
        assert set(a) <= {-1, 0, 1}


def test_crafted_table_emits_wanted_words_in_both_representations():
    """The crafting used by tests/test_gpu_rng_corner_cases.py: words 0..8 zero, words
    397..404 = untempered wanted outputs -> the next eight draws are the wanted outputs, both
    for the block twist at position 624 (oracle / std::mt19937) and for the chunk-wise
    regeneration at mt_idx = 0 (device model), and the two keep agreeing afterwards."""
    import ctypes

    from oracle import oracle_lib
    from toy_text_cases import crafted_table

    L = oracle_lib.lib()
    L.epo_debug_set_rng.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    rng = np.random.default_rng(9)
    orc = oracle_lib.OraclePool("CartPole", 1, seed=0, max_episode_steps=500)
    for _ in range(10):
        want = [int(x) for x in rng.integers(0, 2**32, size=8)]
        want[int(rng.integers(0, 8))] = 0
        want[int(rng.integers(0, 8))] = 0xFFFFFFFF
        mt = crafted_table(rng, want)
        L.epo_debug_set_rng(orc.h, 0, mt.ctypes.data, 624)
        dev = ChunkedMt(0)
        dev.table = mt.copy().reshape(N // 8, 8)
        dev.idx = 0
        got_o = [orc.draw(0) for _ in range(8 + 700)]
        got_d = [dev.next() for _ in range(8 + 700)]
        assert got_o[:8] == want and got_d[:8] == want
        assert got_o == got_d
