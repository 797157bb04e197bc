// Jumanji family: Game2048-v1 and Minesweeper-v0, bit-exact with the reference
// (jumanji/game2048_env.h, jumanji/minesweeper_env.h) including the libstdc++ mt19937
// distribution semantics of Game2048's random cell and Minesweeper's std::shuffle.  One CUDA
// thread per env.  Game2048 first; Minesweeper's layout is described above its struct.
//
// State: the 16 tile exponents (0 = empty) at 5 bits each -- cell c = row * 4 + col lives in
// word c / 6 at bit 5 * (c % 6) -- plus the action mask of the board in bits 20..23 of word 2.
// Exponents stay <= 30: configured cells are at most 26 (game2048_config), and sixteen tiles of
// 2^26 merge into one tile of 2^30 at most, so 5 bits hold every reachable tile.
//
// Each step computes the four directions once, for the board it leaves behind: that gives the
// action mask (written out, and stored in the state) and `done` (no direction moves).  The next
// step reads whether its action moves the board from the stored mask instead of recomputing it.
//
// The pool's configured boards (game2048_initial_board, game2048_replay_boards) sit in the
// state blob where real-valued envs keep rstate, packed like the state: words 0..2 the initial
// board, words 3 + 3 k .. 5 + 3 k replay board k (game2048_config below).  iopt bit 0 is
// add_random_cell, bit 1 "an initial board is configured", bit 2 "replay boards are configured".
#include <cstring>

#include "common.cuh"

namespace epb {

struct Game2048 {
  using Act = int32_t;
  struct State { int32_t w0, w1, w2; };
  static constexpr bool kRngInReset = true, kRngInStep = true, kBlockObs = false;
  static constexpr bool kResetDone = true;  // a configured board may have no legal move
  static constexpr int kReplaySteps = 32;
  static constexpr int kConfigWords = 3 + 3 * kReplaySteps, kMaxConfigCell = 26;

  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    const int64_t n = sv.n_envs;
    s.w0 = sv.istate[e];
    s.w1 = sv.istate[n + e];
    s.w2 = sv.istate[2 * n + e];
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    const int64_t n = sv.n_envs;
    sv.istate[e] = s.w0;
    sv.istate[n + e] = s.w1;
    sv.istate[2 * n + e] = s.w2;
  }
  static __device__ __forceinline__ const int32_t* config(const StateView& sv) {
    return static_cast<const int32_t*>(sv.rstate);
  }

  static __device__ __forceinline__ void unpack(int32_t w0, int32_t w1, int32_t w2, int (&b)[16]) {
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const uint32_t w = (uint32_t)(c < 6 ? w0 : (c < 12 ? w1 : w2));
      b[c] = (int)((w >> (5 * (c % 6))) & 31u);
    }
  }
  static __device__ __forceinline__ void pack(const int (&b)[16], int mask, State& s) {
    uint32_t w[3] = {0u, 0u, 0u};
#pragma unroll
    for (int c = 0; c < 16; ++c) w[c / 6] |= (uint32_t)b[c] << (5 * (c % 6));
    s.w0 = (int32_t)w[0];
    s.w1 = (int32_t)w[1];
    s.w2 = (int32_t)(w[2] | ((uint32_t)mask << 20));
  }
  static __device__ __forceinline__ int mask_of(const State& s) {
    return ((uint32_t)s.w2 >> 20) & 15;
  }

  // Cell of line i, position j (j = 0 is where tiles slide to) for direction A
  // (game2048::Move: 0 up, 1 right, 2 down, 3 left).
  template <int A>
  static __device__ __forceinline__ constexpr int cell(int i, int j) {
    return A == 0 ? j * 4 + i : A == 1 ? i * 4 + (3 - j) : A == 2 ? (3 - j) * 4 + i : i * 4 + j;
  }

  // Whether sliding the line towards position 0 changes it: a tile behind an empty cell, or two
  // equal neighbours once the line is compacted (a line with no tile behind a gap is compacted).
  static __device__ __forceinline__ bool line_moves(int l0, int l1, int l2, int l3) {
    return (l0 == 0 && l1 != 0) || (l1 == 0 && l2 != 0) || (l2 == 0 && l3 != 0) ||
           (l0 != 0 && l0 == l1) || (l1 != 0 && l1 == l2) || (l2 != 0 && l2 == l3);
  }
  template <int A>
  static __device__ __forceinline__ bool moves(const int (&b)[16]) {
    bool m = false;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      m |= line_moves(b[cell<A>(i, 0)], b[cell<A>(i, 1)], b[cell<A>(i, 2)], b[cell<A>(i, 3)]);
    return m;
  }
  static __device__ __forceinline__ int action_mask(const int (&b)[16]) {
    return (moves<0>(b) ? 1 : 0) | (moves<1>(b) ? 2 : 0) | (moves<2>(b) ? 4 : 0) |
           (moves<3>(b) ? 8 : 0);
  }

  static __device__ __forceinline__ float pow2f(int e) {  // ldexp(1.0f, e), 1 <= e <= 31
    return __int_as_float((127 + e) << 23);
  }
  // game2048::MoveLineLeft: compact, then merge equal neighbours left to right; returns the
  // line's reward summed in merge order.
  static __device__ __forceinline__ float slide_line(int& l0, int& l1, int& l2, int& l3) {
    int c[4] = {0, 0, 0, 0};
    int n = 0;
    const int in[4] = {l0, l1, l2, l3};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int k = 0; k < 4; ++k) c[k] = (in[j] != 0 && n == k) ? in[j] : c[k];
      n += in[j] != 0;
    }
    // c[k] != 0 for k < n and 0 beyond, so "c[i] == c[i+1], both tiles" is c[i] != 0 && equal
    float r = 0.0f;
    if (c[0] != 0 && c[0] == c[1]) {
      l0 = c[0] + 1;
      r = __fadd_rn(r, pow2f(l0));
      if (c[2] != 0 && c[2] == c[3]) {
        l1 = c[2] + 1;
        r = __fadd_rn(r, pow2f(l1));
        l2 = 0;
      } else {
        l1 = c[2];
        l2 = c[3];
      }
      l3 = 0;
    } else {
      l0 = c[0];
      if (c[1] != 0 && c[1] == c[2]) {
        l1 = c[1] + 1;
        r = __fadd_rn(r, pow2f(l1));
        l2 = c[3];
        l3 = 0;
      } else {
        l1 = c[1];
        if (c[2] != 0 && c[2] == c[3]) {
          l2 = c[2] + 1;
          r = __fadd_rn(r, pow2f(l2));
          l3 = 0;
        } else {
          l2 = c[2];
          l3 = c[3];
        }
      }
    }
    return r;
  }
  // game2048::Move: lines i = 0..3, their rewards added in that order
  template <int A>
  static __device__ __forceinline__ float move(int (&b)[16]) {
    float r = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      r = __fadd_rn(r, slide_line(b[cell<A>(i, 0)], b[cell<A>(i, 1)], b[cell<A>(i, 2)],
                                  b[cell<A>(i, 3)]));
    return r;
  }

  // Game2048Env::AddRandomCell: `board_[empty[position_dist(gen_)]] = two_dist(gen_) ? 2 : 1;`
  // Under C++17 the right-hand side is sequenced first, so the bernoulli_distribution(0.1) draw
  // (generate_canonical<double>: 2 words, compared < 0.1) precedes the
  // uniform_int_distribution(0, n_empty - 1) draw (Lemire: 1 word plus rejections).
  static __device__ __forceinline__ void add_random_cell(int (&b)[16], Mt* rng) {
    int n = 0;
#pragma unroll
    for (int c = 0; c < 16; ++c) n += b[c] == 0;
    if (n == 0) return;
    const int value = rng->canonical() < 0.1 ? 2 : 1;
    const int k = rng->uniform_int(0, n - 1);
    int seen = 0;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const bool empty = b[c] == 0;
      b[c] = (empty && seen == k) ? value : b[c];
      seen += empty;
    }
  }

  static __device__ __forceinline__ void reset(const StateView& sv, State& s, Mt* rng,
                                               StepOut& so, int& done) {
    int b[16];
    if (sv.iopt & 2) {
      const int32_t* cfg = config(sv);
      unpack(cfg[0], cfg[1], cfg[2], b);
    } else {
#pragma unroll
      for (int c = 0; c < 16; ++c) b[c] = 0;
      add_random_cell(b, rng);
    }
    const int mask = action_mask(b);
    done = mask == 0;
    pack(b, mask, s);
    so.reward = 0.0f;
  }

  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt* rng, StepOut& so) {
    const int a = act < 0 ? 0 : (act > 3 ? 3 : act);
    int b[16];
    unpack(s.w0, s.w1, s.w2, b);
    float reward = 0.0f;
    if ((mask_of(s) >> a) & 1) {
      switch (a) {
        case 0: reward = move<0>(b); break;
        case 1: reward = move<1>(b); break;
        case 2: reward = move<2>(b); break;
        default: reward = move<3>(b); break;
      }
      if (sv.iopt & 1) add_random_cell(b, rng);
    }
    if ((sv.iopt & 4) && cur <= kReplaySteps) {
      const int32_t* r = config(sv) + 3 * cur;  // replay board cur - 1 starts at word 3 * cur
      unpack(r[0], r[1], r[2], b);
    }
    const int mask = action_mask(b);
    done = mask == 0;
    pack(b, mask, s);
    so.reward = reward;
  }

  static __device__ __forceinline__ void write_obs(const StateView&, const OutView& ov,
                                                   int64_t row, const State& s, const StepOut&) {
    int b[16];
    unpack(s.w0, s.w1, s.w2, b);
    int hi = 0;
#pragma unroll
    for (int c = 0; c < 16; ++c) hi = b[c] > hi ? b[c] : hi;
    if (ov.env[0]) {
      int4* o = reinterpret_cast<int4*>(static_cast<int32_t*>(ov.env[0]) + row * 16);
#pragma unroll
      for (int r = 0; r < 4; ++r)
        o[r] = make_int4(b[4 * r], b[4 * r + 1], b[4 * r + 2], b[4 * r + 3]);
    }
    if (ov.env[1]) {
      const int m = mask_of(s);
      static_cast<uchar4*>(ov.env[1])[row] =
          make_uchar4(m & 1, (m >> 1) & 1, (m >> 2) & 1, (m >> 3) & 1);
    }
    if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[row] = hi == 0 ? 1 : (1 << hi);
  }
};

// ------------------------------------------------------------------------------ Minesweeper
// Minesweeper-v0 (jumanji/minesweeper_env.h), 10 x 10 cells, cell c = row * 10 + col.
//
// State, 17 istate words:
//   words 0..12  the board, cell c at bits 4 * (c % 8) of word c / 8 as value + 1 (0 = unexplored,
//                1..9 = 0..8 adjacent mines); bits 16..31 of word 12 hold step_count
//   words 13..16 the mine mask, cell c at bit c % 32 of word 13 + c / 32
// The board is stored, not derived from the mines: replay boards overwrite it with any cells.
//
// The step works on 100-bit bitboards (Bb: cells 0..63 in lo, 64..99 in hi).  Adjacent-mine
// counts are four bit planes summed from the eight shifted mine masks.  Reveal (a BFS in the
// reference) is a fixed point: the clicked cell's 8-connected component inside {unexplored,
// no mine, count 0}, grown by one dilation per round; the cells revealed are that component
// dilated once (or the clicked cell alone), intersected with the unexplored cells.  That set
// does not depend on the BFS order.
//
// The pool's configuration sits in the state blob where real-valued envs keep rstate
// (minesweeper_config below): word 0 flags (bit 0: mines are configured, bit 1: replay is on), words
// 1..4 the configured mine mask, 5 + 13 k .. 17 + 13 k replay board k packed as the state's words
// 0..12, 421 + k replay reward k (float bits), 453 the replay done flags (bit k).  The flags live
// there, not in iopt, so that a state snapshot carries the whole configuration.
struct Bb {
  uint64_t lo, hi;
};
__device__ __forceinline__ Bb operator&(Bb a, Bb b) { return {a.lo & b.lo, a.hi & b.hi}; }
__device__ __forceinline__ Bb operator|(Bb a, Bb b) { return {a.lo | b.lo, a.hi | b.hi}; }
__device__ __forceinline__ Bb operator^(Bb a, Bb b) { return {a.lo ^ b.lo, a.hi ^ b.hi}; }
__device__ __forceinline__ Bb operator~(Bb a) { return {~a.lo, ~a.hi}; }

struct Minesweeper {
  using Act = ActI32x2;
  struct State {
    uint32_t b[13];  // board nibbles (+ step_count in b[12] >> 16)
    uint32_t m[4];   // mine mask
  };
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = true;
  static constexpr int kW = 10, kCells = 100, kBoardWords = 13, kMineWords = 4;
  static constexpr int kDefaultMines = 10, kReplaySteps = 32;
  static constexpr int kCfgMines = 1, kCfgReplay = 5, kCfgRewards = kCfgReplay + 13 * 32,
                       kCfgDone = kCfgRewards + 32, kConfigWords = kCfgDone + 1;

  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    const int64_t n = sv.n_envs;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < kBoardWords; ++k) s.b[k] = w[k * n + e];
#pragma unroll
    for (int k = 0; k < kMineWords; ++k) s.m[k] = w[(kBoardWords + k) * n + e];
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    const int64_t n = sv.n_envs;
    uint32_t* w = reinterpret_cast<uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < kBoardWords; ++k) w[k * n + e] = s.b[k];
#pragma unroll
    for (int k = 0; k < kMineWords; ++k) w[(kBoardWords + k) * n + e] = s.m[k];
  }
  static __device__ __forceinline__ const uint32_t* config(const StateView& sv) {
    return static_cast<const uint32_t*>(sv.rstate);
  }

  // ---- bitboards
  static __device__ __forceinline__ constexpr uint64_t col_bits(int c, int base) {
    uint64_t v = 0;
    for (int i = 0; i < 64; ++i)
      if (base + i < kCells && (base + i) % kW == c) v |= 1ull << i;
    return v;
  }
  static constexpr uint64_t kAllHi = (1ull << (kCells - 64)) - 1;
  template <int K>
  static __device__ __forceinline__ Bb shl(Bb x) {  // cell c -> c + K, clipped to the board
    return {x.lo << K, ((x.hi << K) | (x.lo >> (64 - K))) & kAllHi};
  }
  template <int K>
  static __device__ __forceinline__ Bb shr(Bb x) {  // cell c -> c - K
    return {(x.lo >> K) | (x.hi << (64 - K)), x.hi >> K};
  }
  // cell c gets cell c + 1 / c - 1 of its own row (0 past the edge)
  static __device__ __forceinline__ Bb from_right(Bb x) {
    return shr<1>(x) & Bb{~col_bits(kW - 1, 0), ~col_bits(kW - 1, 64)};
  }
  static __device__ __forceinline__ Bb from_left(Bb x) {
    return shl<1>(x) & Bb{~col_bits(0, 0), ~col_bits(0, 64)};
  }
  // x and its 8 neighbours
  static __device__ __forceinline__ Bb dilate(Bb x) {
    const Bb h = x | from_right(x) | from_left(x);
    return h | shr<kW>(h) | shl<kW>(h);
  }
  static __device__ __forceinline__ bool same(Bb a, Bb b) { return a.lo == b.lo && a.hi == b.hi; }
  static __device__ __forceinline__ Bb cell_bit(int c) {
    return {c < 64 ? 1ull << c : 0ull, c >= 64 ? 1ull << (c - 64) : 0ull};
  }
  static __device__ __forceinline__ Bb mines_of(const State& s) {
    return {(uint64_t)s.m[0] | ((uint64_t)s.m[1] << 32),
            (uint64_t)s.m[2] | ((uint64_t)s.m[3] << 32)};
  }
  // byte k (cells 8k .. 8k + 7) of a bitboard
  static __device__ __forceinline__ uint32_t byte_of(Bb x, int k) {
    return (uint32_t)((k < 8 ? x.lo >> (8 * k) : x.hi >> (8 * (k - 8))) & 0xffu);
  }
  // 8 bits <-> one bit per nibble (bit j <-> bit 4 j)
  static __device__ __forceinline__ uint32_t spread8(uint32_t x) {
    x = (x | (x << 12)) & 0x000f000fu;
    x = (x | (x << 6)) & 0x03030303u;
    return (x | (x << 3)) & 0x11111111u;
  }
  static __device__ __forceinline__ uint32_t gather8(uint32_t x) {
    x = (x | (x >> 3)) & 0x03030303u;
    x = (x | (x >> 6)) & 0x000f000fu;
    return (x | (x >> 12)) & 0xffu;
  }
  // bit 4 j set where nibble j is 0 (an unexplored cell)
  static __device__ __forceinline__ uint32_t zero_nibbles(uint32_t w) {
    return ~(w | (w >> 1) | (w >> 2) | (w >> 3)) & 0x11111111u;
  }
  static __device__ __forceinline__ Bb unexplored(const State& s) {
    Bb u{0ull, 0ull};
#pragma unroll
    for (int k = 0; k < kBoardWords; ++k) {
      const uint64_t z = gather8(zero_nibbles(k == 12 ? (s.b[k] | 0xffff0000u) : s.b[k]));
      if (k < 8) u.lo |= z << (8 * k);
      else u.hi |= z << (8 * (k - 8));
    }
    return u;
  }
  // c[0..3] += x, bit-sliced
  static __device__ __forceinline__ void add1(Bb (&c)[4], Bb x) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const Bb carry = c[k] & x;
      c[k] = c[k] ^ x;
      x = carry;
    }
  }

  // MinesweeperEnv::Reveal of a valid click on unexplored `cell`: writes the revealed cells'
  // adjacent-mine counts into the board and returns the cells still unexplored.
  static __device__ __forceinline__ Bb reveal(State& s, Bb mines, Bb unexp, int cell) {
    Bb cnt[4] = {{0ull, 0ull}, {0ull, 0ull}, {0ull, 0ull}, {0ull, 0ull}};
    const Bb r = from_right(mines), l = from_left(mines);
    add1(cnt, r);
    add1(cnt, l);
    add1(cnt, shl<kW>(mines));  // the row above
    add1(cnt, shl<kW>(r));
    add1(cnt, shl<kW>(l));
    add1(cnt, shr<kW>(mines));  // the row below
    add1(cnt, shr<kW>(r));
    add1(cnt, shr<kW>(l));
    const Bb zero = unexp & ~mines & ~(cnt[0] | cnt[1] | cnt[2] | cnt[3]);
    const Bb seed = cell_bit(cell);
    Bb comp = seed & zero;
#pragma unroll 1
    while (true) {
      const Bb next = dilate(comp) & zero;
      if (same(next, comp)) break;
      comp = next;
    }
    const Bb rev = (dilate(comp) | seed) & unexp;
#pragma unroll
    for (int k = 0; k < kBoardWords; ++k) {
      const uint32_t sel = spread8(byte_of(rev, k)) * 0xfu;
      const uint32_t val = (spread8(byte_of(cnt[0], k)) | (spread8(byte_of(cnt[1], k)) << 1) |
                            (spread8(byte_of(cnt[2], k)) << 2) |
                            (spread8(byte_of(cnt[3], k)) << 3)) + 0x11111111u;
      s.b[k] = (s.b[k] & ~sel) | (val & sel);
    }
    return unexp & ~rev;
  }
  static __device__ __forceinline__ int popc(Bb x) { return __popcll(x.lo) + __popcll(x.hi); }
  static __device__ __forceinline__ bool bit(Bb x, int c) {
    return ((c < 64 ? x.lo >> c : x.hi >> (c - 64)) & 1ull) != 0;
  }
  // std::iter_swap(front + a, front + b) on the tracked front positions, a a constant
  static __device__ __forceinline__ void swap_front(int (&f)[kDefaultMines], int a, int b) {
    const int va = f[a];
    int vb = f[0];
#pragma unroll
    for (int q = 1; q < kDefaultMines; ++q) vb = q == b ? f[q] : vb;
    f[a] = vb;
#pragma unroll
    for (int q = 0; q < kDefaultMines; ++q) f[q] = q == b ? va : f[q];
  }
  // The first 10 cells of std::shuffle(iota(100), gen_) (libstdc++ 13 bits/stl_algo.h): one
  // uniform_int{0, 1} for position 1, then position pairs (i, i + 1), i = 2, 4, .., 98, from
  // one uniform_int{0, (i + 1)(i + 2) - 1} draw x each: swap i with x / (i + 2), then i + 1
  // with x % (i + 2).  Before its own swap position i still holds i (earlier swaps touch only
  // positions <= their step), so for i >= 10 a swap with a front position j just sets
  // front[j] = i and the other 90 positions need no storage.
  static __device__ __forceinline__ Bb random_mines(Mt& rng) {
    int f[kDefaultMines];
#pragma unroll
    for (int q = 0; q < kDefaultMines; ++q) f[q] = q;
    swap_front(f, 1, rng.uniform_int(0, 1));
#pragma unroll
    for (int i = 2; i < kDefaultMines; i += 2) {
      const uint32_t x = (uint32_t)rng.uniform_int(0, (i + 1) * (i + 2) - 1);
      swap_front(f, i, (int)(x / (i + 2)));
      swap_front(f, i + 1, (int)(x % (i + 2)));
    }
#pragma unroll 1
    for (int i = kDefaultMines; i < kCells; i += 2) {
      const uint32_t x = (uint32_t)rng.uniform_int(0, (i + 1) * (i + 2) - 1);
      const int j = (int)(x / (uint32_t)(i + 2)), k = (int)(x % (uint32_t)(i + 2));
#pragma unroll
      for (int q = 0; q < kDefaultMines; ++q) f[q] = q == j ? i : f[q];
#pragma unroll
      for (int q = 0; q < kDefaultMines; ++q) f[q] = q == k ? i + 1 : f[q];
    }
    Bb m{0ull, 0ull};
#pragma unroll
    for (int q = 0; q < kDefaultMines; ++q) m = m | cell_bit(f[q]);
    return m;
  }

  static __device__ __forceinline__ void reset(const StateView& sv, State& s, Mt* rng,
                                               StepOut& so) {
#pragma unroll
    for (int k = 0; k < kBoardWords; ++k) s.b[k] = 0u;  // all unexplored, step_count 0
    const uint32_t* cfg = config(sv);
    if (cfg[0] & 1u) {
#pragma unroll
      for (int k = 0; k < kMineWords; ++k) s.m[k] = cfg[kCfgMines + k];
    } else {
      const Bb m = random_mines(*rng);
      s.m[0] = (uint32_t)m.lo;
      s.m[1] = (uint32_t)(m.lo >> 32);
      s.m[2] = (uint32_t)m.hi;
      s.m[3] = (uint32_t)(m.hi >> 32);
    }
    so.reward = 0.0f;
  }

  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt*, StepOut& so) {
    float reward = 0.0f;
    const uint32_t* cfg = config(sv);
    if ((cfg[0] & 2u) && cur <= kReplaySteps) {  // the replay ignores the action
      const uint32_t* board = cfg + kCfgReplay + kBoardWords * (cur - 1);
#pragma unroll
      for (int k = 0; k < kBoardWords; ++k) s.b[k] = board[k];
      reward = __uint_as_float(cfg[kCfgRewards + cur - 1]);
      done = (cfg[kCfgDone] >> (cur - 1)) & 1u;
    } else {
      const int row = act.x < 0 ? 0 : (act.x > kW - 1 ? kW - 1 : act.x);
      const int col = act.y < 0 ? 0 : (act.y > kW - 1 ? kW - 1 : act.y);
      const int cell = row * kW + col;
      const Bb mines = mines_of(s), unexp = unexplored(s);
      const bool valid = bit(unexp, cell), hit = bit(mines, cell);
      bool solved = false;
      if (valid) {
        // explored == 100 - num_mines  <=>  unexplored == num_mines
        solved = popc(reveal(s, mines, unexp, cell)) == popc(mines);
        reward = hit ? 0.0f : 1.0f;
      }
      done = !valid || hit || solved;
    }
    s.b[kBoardWords - 1] = (s.b[kBoardWords - 1] & 0xffffu) | ((uint32_t)cur << 16);
    so.reward = reward;
  }

  // obs:num_mines and obs:step_count are one coalesced 4-byte store per thread.  The 400 B
  // obs:board and 100 B obs:action_mask rows would be 400 B / 100 B apart across a warp's
  // lanes, so the CTA stages its envs' board words in shared memory and writes rows
  // [row0, min(row0 + kB, row_end)) of both columns as contiguous runs: 16-byte board chunks
  // and 4-byte mask words, four cells each (one 16-bit half of a board word).
  template <int kB>
  static __device__ __forceinline__ void block_write_obs(const OutView& ov, int64_t row0,
                                                         int64_t row_end, bool active,
                                                         const State& s, const StepOut&) {
    // [env][word]: 13 is odd, so the staging stores of a warp hit 32 different banks
    __shared__ uint32_t sb[kB][kBoardWords];
    if (active) {
      const int64_t row = row0 + threadIdx.x;
#pragma unroll
      for (int k = 0; k < kBoardWords; ++k) sb[threadIdx.x][k] = s.b[k];
      if (ov.env[2])
        static_cast<int32_t*>(ov.env[2])[row] =
            __popc(s.m[0]) + __popc(s.m[1]) + __popc(s.m[2]) + __popc(s.m[3]);
      if (ov.env[3]) static_cast<int32_t*>(ov.env[3])[row] = (int)(s.b[kBoardWords - 1] >> 16);
    }
    __syncthreads();
    int64_t rows = row_end - row0;
    if (rows > kB) rows = kB;
    constexpr int kChunks = kCells / 4;  // per row
    const int nvec = (int)rows * kChunks;
    int4* board = ov.env[0] ? reinterpret_cast<int4*>(static_cast<int32_t*>(ov.env[0]) +
                                                      row0 * kCells)
                            : nullptr;
    uint32_t* mask = ov.env[1] ? reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(ov.env[1]) +
                                                             row0 * kCells)
                               : nullptr;
    for (int v = threadIdx.x; v < nvec; v += kB) {
      const int e = v / kChunks, j = v - e * kChunks;
      const uint32_t h = sb[e][j >> 1] >> (16 * (j & 1));
      const uint32_t n0 = h & 15u, n1 = (h >> 4) & 15u, n2 = (h >> 8) & 15u, n3 = (h >> 12) & 15u;
      if (board) board[v] = make_int4((int)n0 - 1, (int)n1 - 1, (int)n2 - 1, (int)n3 - 1);
      if (mask)
        mask[v] = (n0 == 0u ? 1u : 0u) | (n1 == 0u ? 1u << 8 : 0u) | (n2 == 0u ? 1u << 16 : 0u) |
                  (n3 == 0u ? 1u << 24 : 0u);
    }
    __syncthreads();
  }
};

const char* game2048_config(const int32_t* initial16, const int32_t* replay512,
                            std::vector<uint32_t>& words, int32_t& iopt) {
  auto check = [](const int32_t* v, int n) {
    for (int i = 0; i < n; ++i)
      if (v[i] < 0 || v[i] > Game2048::kMaxConfigCell) return false;
    return true;
  };
  if ((initial16 && !check(initial16, 16)) || (replay512 && !check(replay512, 16 * 32)))
    return "Game2048 board cells must be tile exponents in [0, 26]";
  words.assign(Game2048::kConfigWords, 0u);
  auto pack = [](const int32_t* b, uint32_t* w) {
    for (int c = 0; c < 16; ++c) w[c / 6] |= (uint32_t)b[c] << (5 * (c % 6));
  };
  if (initial16) pack(initial16, words.data());
  for (int k = 0; replay512 && k < Game2048::kReplaySteps; ++k)
    pack(replay512 + 16 * k, words.data() + 3 + 3 * k);
  iopt = (iopt & 1) | (initial16 ? 2 : 0) | (replay512 ? 4 : 0);
  return nullptr;
}

const char* minesweeper_config(const int32_t* mines100, const int32_t* replay_boards3200,
                               const float* replay_rewards32, const uint8_t* replay_done32,
                               std::vector<uint32_t>& words) {
  using M = Minesweeper;
  // the kernel stores value + 1 in 4 bits: -1 (unexplored) .. 8 adjacent mines
  for (int i = 0; replay_boards3200 && i < M::kReplaySteps * M::kCells; ++i)
    if (replay_boards3200[i] < -1 || replay_boards3200[i] > 8)
      return "Minesweeper replay board cells must lie in [-1, 8]";
  words.assign(M::kConfigWords, 0u);
  for (int c = 0; mines100 && c < M::kCells; ++c)
    if (mines100[c]) {
      words[M::kCfgMines + c / 32] |= 1u << (c % 32);
      words[0] |= 1u;  // at least one mine: configured placement
    }
  if (replay_boards3200) words[0] |= 2u;
  for (int k = 0; replay_boards3200 && k < M::kReplaySteps; ++k) {
    for (int c = 0; c < M::kCells; ++c)
      words[M::kCfgReplay + M::kBoardWords * k + c / 8] |=
          (uint32_t)(replay_boards3200[M::kCells * k + c] + 1) << (4 * (c % 8));
    if (replay_rewards32) std::memcpy(&words[M::kCfgRewards + k], &replay_rewards32[k], 4);
    if (replay_done32 && replay_done32[k]) words[M::kCfgDone] |= 1u << k;
  }
  return nullptr;
}

// The entries' order is the order in which the kernels are instantiated, and the code ptxas
// makes for Minesweeper's 128-thread step kernel depends on it: reordering them changes SASS.
const KindDesc kJumanjiKinds[] = {
    // jumanji/minesweeper_env.h MinesweeperEnvFns.  No options: minesweeper_config configures.
    // Draws only at reset (50 words): like the classic envs' reset draws, not counted.
    {.kind = EPB_MINESWEEPER,
     .keys = {{"obs:board", EPB_I32, 2, {Minesweeper::kW, Minesweeper::kW}},
              {"obs:action_mask", EPB_BOOL, 2, {Minesweeper::kW, Minesweeper::kW}},
              {"obs:num_mines", EPB_I32, 0, {}}, {"obs:step_count", EPB_I32, 0, {}}},
     .action = {"action", EPB_I32, 1, {2}},  // (row, column)
     .NI = Minesweeper::kBoardWords + Minesweeper::kMineWords,
     .config_words = Minesweeper::kConfigWords, .iopts = {0}, .n_iopts = 1,
     .iopt_error = "Minesweeper iopt must be -1 or 0", .launch = fixed_launch<Minesweeper>},
    // jumanji/game2048_env.h Game2048EnvFns::StateSpec; iopt: add_random_cell
    {.kind = EPB_GAME2048,
     .keys = {{"obs:board", EPB_I32, 2, {4, 4}}, {"obs:action_mask", EPB_BOOL, 1, {4}},
              {"info:highest_tile", EPB_I32, 0, {}}},
     .action = kDiscreteAction, .NI = kStateWords<Game2048>,
     .config_words = Game2048::kConfigWords, .default_iopt = 1, .iopts = {0, 1}, .n_iopts = 2,
     .iopt_error = "Game2048 iopt (add_random_cell) must be -1, 0 or 1",
     // 3 words per moving step (bernoulli 2, Lemire 1)
     .launch = fixed_launch<Game2048, 3 * 16 + 8>},
};
const KindDesc* jumanji_kind(int kind) { return find_kind(kJumanjiKinds, kind); }

}  // namespace epb
