// PGX family: TicTacToe-v1, ConnectFour-v1, Hex-v1 and Othello-v1 (pgx/board_games.h
// TicTacToeEnv, ConnectFourEnv, HexEnv, OthelloEnv), bit-exact with the reference.  The engine's first two-player kinds: every env row has two
// player rows in the per-player columns (obs, info:players.id and the common
// info:players.env_id, reward and discount; common.cuh write_common_pair).  One CUDA thread
// per env.
//
// State: the board as one bitboard per colour, colour c's stones in b[c], plus flags -- bit 0
// color_ (the colour to move), bit 1 current_player_ (the player to move), bit 2 "the last step
// ended the game" (the legal-action mask then reads all true).  Player p plays colour
// p ^ (current_player_ != color_); a step flips both bits, so that relation holds for the whole
// episode and is what PlayerRewards and WriteObservation compute.
//   TicTacToe    cell c = row * 3 + col at bit c; one istate word: b[0] bits 0..8, b[1] bits
//                9..17, flags bits 18..20
//   ConnectFour  cell (row, col), row 0 at the top, at bit 7 col + 5 - row: each column is 7
//                bits, bottom stone first, the 7th bit always empty -- so a win is four of one
//                colour along a shift of 1 (vertical), 7 (horizontal), 6 or 8 (the diagonals),
//                and no shift wraps across the board's edge.  Five istate words: b[0] lo, hi,
//                b[1] lo, hi, flags
// The win tests look at the whole board of the colour that moved, as the reference's
// StepGame / HasWon scans do.
//
// Reset draws one mt19937 word (current_player_ = gen_() & 1) and nothing else draws.  Bytes per
// env-step (identity batch, epb_bytes_per_env_step): TicTacToe 151 = 4 action + 2 x (4 flags +
// 4 state) + 38 common columns (two player rows of info:players.env_id, reward, discount) + 93
// env columns (36 obs, 36 info:board, 4 info:current_player, 9 info:legal_action_mask,
// 8 info:players.id); ConnectFour 445 = 4 + 2 x (4 + 20) + 38 + 355 (168, 168, 4, 7, 8); Hex
// 1708 = 4 + 2 x (4 + 36) + 38 + 1586 (968, 484, 4, 122, 8); Othello 679 = 4 + 2 x (4 + 20) + 38 +
// 589 (256, 256, 4, 65, 8).  Hex and Othello have their own Envs below.
#include "common.cuh"

namespace epb {

struct TicTacToeRules {
  static constexpr int kRows = 3, kCols = 3, kActions = 9, kWords = 1;
  static __device__ __forceinline__ int bit_of(int cell) { return cell; }
  static __device__ __forceinline__ bool playable(uint64_t occ, int a) {
    return ((occ >> a) & 1ull) == 0ull;
  }
  // an in-range move overwrites its cell, occupied or not (StepGame)
  static __device__ __forceinline__ uint64_t move_bit(uint64_t, int a) { return 1ull << a; }
  static __device__ __forceinline__ bool won(uint64_t x) {
    constexpr uint32_t kLines[8] = {0x007u, 0x038u, 0x1c0u, 0x049u,
                                    0x092u, 0x124u, 0x111u, 0x054u};
    const uint32_t b = (uint32_t)x;
    bool w = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) w |= (b & kLines[k]) == kLines[k];
    return w;
  }
  static __device__ __forceinline__ bool full(uint64_t occ) { return occ == 0x1ffull; }
  static __device__ __forceinline__ void load(const uint32_t (&w)[kWords], uint64_t (&b)[2],
                                              uint32_t& f) {
    b[0] = w[0] & 0x1ffu;
    b[1] = (w[0] >> 9) & 0x1ffu;
    f = w[0] >> 18;
  }
  static __device__ __forceinline__ void store(uint32_t (&w)[kWords], const uint64_t (&b)[2],
                                               uint32_t f) {
    w[0] = (uint32_t)b[0] | ((uint32_t)b[1] << 9) | (f << 18);
  }
};

struct ConnectFourRules {
  static constexpr int kRows = 6, kCols = 7, kActions = 7, kWords = 5;
  static constexpr uint64_t kFull = 0x3full | 0x3full << 7 | 0x3full << 14 | 0x3full << 21 |
                                    0x3full << 28 | 0x3full << 35 | 0x3full << 42;
  static __device__ __forceinline__ int bit_of(int cell) {
    const int row = cell / kCols, col = cell - row * kCols;
    return 7 * col + 5 - row;
  }
  // a column takes a stone while its top cell is empty (columns fill from the bottom)
  static __device__ __forceinline__ bool playable(uint64_t occ, int a) {
    return ((occ >> (7 * a + 5)) & 1ull) == 0ull;
  }
  // the lowest empty cell of column a; a full column takes nothing (StepGame, row < 0)
  static __device__ __forceinline__ uint64_t move_bit(uint64_t occ, int a) {
    const int h = __popcll((occ >> (7 * a)) & 0x3full);
    return h < 6 ? 1ull << (7 * a + h) : 0ull;
  }
  static __device__ __forceinline__ bool won(uint64_t x) {
    constexpr int kShifts[4] = {1, 7, 6, 8};  // vertical, horizontal, the two diagonals
    bool w = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t m = x & (x >> kShifts[k]);
      w |= (m & (m >> (2 * kShifts[k]))) != 0ull;
    }
    return w;
  }
  static __device__ __forceinline__ bool full(uint64_t occ) { return occ == kFull; }
  static __device__ __forceinline__ void load(const uint32_t (&w)[kWords], uint64_t (&b)[2],
                                              uint32_t& f) {
    b[0] = (uint64_t)w[0] | ((uint64_t)w[1] << 32);
    b[1] = (uint64_t)w[2] | ((uint64_t)w[3] << 32);
    f = w[4];
  }
  static __device__ __forceinline__ void store(uint32_t (&w)[kWords], const uint64_t (&b)[2],
                                               uint32_t f) {
    w[0] = (uint32_t)b[0];
    w[1] = (uint32_t)(b[0] >> 32);
    w[2] = (uint32_t)b[1];
    w[3] = (uint32_t)(b[1] >> 32);
    w[4] = f;
  }
};

template <class R>
struct BoardGame {
  using Act = int32_t;
  struct State {
    uint32_t w[R::kWords];
  };
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = true;
  static constexpr int kPlayers = 2;
  static constexpr int kCells = R::kRows * R::kCols;
  static constexpr uint32_t kColor = 1u, kPlayer = 2u, kOver = 4u;

  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    const int64_t n = sv.n_envs;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < R::kWords; ++k) s.w[k] = w[k * n + e];
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    const int64_t n = sv.n_envs;
    uint32_t* w = reinterpret_cast<uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < R::kWords; ++k) w[k * n + e] = s.w[k];
  }

  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    const uint64_t b[2] = {0ull, 0ull};
    R::store(s.w, b, (rng->next() & 1u) ? kPlayer : 0u);  // color_ 0, current_player_ drawn
    so.reward = 0.0f;
    so.extra = 0.0f;
  }

  // TicTacToeEnv::Step / ConnectFourEnv::Step.  The mover is the player to move (the loser of
  // an illegal move, the winner of a winning one): rewards are +-1 for that player and the
  // negation for the other.
  static __device__ __forceinline__ void step(const StateView&, State& s, Act act, int, int& done,
                                              Mt*, StepOut& so) {
    uint64_t b[2];
    uint32_t f;
    R::load(s.w, b, f);
    const int color = (int)(f & kColor);
    const uint32_t mover = (f & kPlayer) ? 1u : 0u;
    const bool in_range = act >= 0 && act < R::kActions;
    const bool illegal = !in_range || !R::playable(b[0] | b[1], act);
    bool won = false;
    if (in_range) {  // StepGame runs for every in-range move, legal or not
      const uint64_t bit = R::move_bit(b[0] | b[1], act);
      const uint64_t mine = (color ? b[1] : b[0]) | bit, theirs = (color ? b[0] : b[1]) & ~bit;
      b[0] = color ? theirs : mine;
      b[1] = color ? mine : theirs;
      won = R::won(mine);
      f ^= kColor | kPlayer;
    }
    float r_mover = 0.0f;
    if (illegal) {
      done = 1;
      r_mover = -1.0f;
    } else {
      done = won || R::full(b[0] | b[1]);
      r_mover = won ? 1.0f : 0.0f;
    }
    f = done ? (f | kOver) : (f & ~kOver);
    R::store(s.w, b, f);
    so.reward = 0.0f;  // players 0 and 1; a draw or a running game gives +0.0f to both
    so.extra = 0.0f;
    if (r_mover != 0.0f) {
      so.reward = mover ? -r_mover : r_mover;
      so.extra = -so.reward;
    }
  }

  // info:current_player and info:players.id are one coalesced store per thread.  obs
  // (2 x 2 x kCells bool), info:board (kCells int32) and info:legal_action_mask (kActions bool)
  // rows would be tens of bytes apart across a warp's lanes, so the CTA stages its envs'
  // states in shared memory and writes rows [row0, min(row0 + kB, row_end)) of each column as
  // one contiguous run: obs in 4-byte words, the board in int32, the mask bytewise.
  template <int kB>
  static __device__ __forceinline__ void block_write_obs(const OutView& ov, int64_t row0,
                                                         int64_t row_end, bool active,
                                                         const State& s, const StepOut&) {
    __shared__ uint64_t sb[2][kB];
    __shared__ uint32_t sf[kB];
    if (active) {
      const int64_t row = row0 + threadIdx.x;
      uint64_t b[2];
      uint32_t f;
      R::load(s.w, b, f);
      sb[0][threadIdx.x] = b[0];
      sb[1][threadIdx.x] = b[1];
      sf[threadIdx.x] = f;
      if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[row] = (f & kPlayer) ? 1 : 0;
      if (ov.env[4]) reinterpret_cast<int2*>(ov.env[4])[row] = make_int2(0, 1);
    }
    __syncthreads();
    int64_t rows = row_end - row0;
    if (rows > kB) rows = kB;
    if (ov.env[0]) {
      // obs[player][row][col][plane]: plane 0 the player's own stones, plane 1 the opponent's
      constexpr int kObsBytes = 2 * kCells * 2;
      uint32_t* obs = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(ov.env[0]) +
                                                  row0 * kObsBytes);
      const int nw = (int)rows * (kObsBytes / 4);
      for (int v = threadIdx.x; v < nw; v += kB) {
        const int e = v / (kObsBytes / 4), k0 = 4 * (v - e * (kObsBytes / 4));
        const uint32_t swap = ((sf[e] >> 1) ^ sf[e]) & 1u;  // current_player_ != color_
        uint32_t word = 0u;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int k = k0 + q;
          const int p = k / (2 * kCells), m = k - p * (2 * kCells);
          const uint32_t c = (uint32_t)p ^ swap ^ (uint32_t)(m & 1);
          word |= (uint32_t)((sb[c][e] >> R::bit_of(m >> 1)) & 1ull) << (8 * q);
        }
        obs[v] = word;
      }
    }
    if (ov.env[1]) {
      int32_t* board = static_cast<int32_t*>(ov.env[1]) + row0 * kCells;
      const int nv = (int)rows * kCells;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v / kCells, bit = R::bit_of(v - e * kCells);
        board[v] = ((sb[0][e] >> bit) & 1ull) ? 0 : (((sb[1][e] >> bit) & 1ull) ? 1 : -1);
      }
    }
    if (ov.env[3]) {
      uint8_t* mask = static_cast<uint8_t*>(ov.env[3]) + row0 * R::kActions;
      const int nv = (int)rows * R::kActions;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v / R::kActions, a = v - e * R::kActions;
        mask[v] = (sf[e] & kOver) || R::playable(sb[0][e] | sb[1][e], a) ? 1 : 0;
      }
    }
    __syncthreads();
  }
};

using TicTacToe = BoardGame<TicTacToeRules>;
using ConnectFour = BoardGame<ConnectFourRules>;

// Hex-v1 and Othello-v1 (board_games.h HexEnv, OthelloEnv).  Their steps, masks and observation
// planes share nothing with BoardGame's, so each is its own Env over the same kind of state: a
// bitboard per side in kWords - 1 istate words (word-major, like BoardGame) and a flags word.
template <int kWords>
struct BitboardState {
  struct State {
    uint32_t w[kWords];
  };
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    const int64_t n = sv.n_envs;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < kWords; ++k) s.w[k] = w[k * n + e];
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    const int64_t n = sv.n_envs;
    uint32_t* w = reinterpret_cast<uint32_t*>(sv.istate);
#pragma unroll
    for (int k = 0; k < kWords; ++k) w[k * n + e] = s.w[k];
  }
};

// A 128-bit board as two 64-bit words (bits 0..63 in lo), with the operators Hex needs; shifts
// take 0 < k < 64.
struct B128 {
  uint64_t lo, hi;
};
__device__ __forceinline__ B128 make_b128(uint64_t hi, uint64_t lo) { return {lo, hi}; }
__device__ __forceinline__ B128 operator|(B128 a, B128 b) { return {a.lo | b.lo, a.hi | b.hi}; }
__device__ __forceinline__ B128 operator&(B128 a, B128 b) { return {a.lo & b.lo, a.hi & b.hi}; }
__device__ __forceinline__ B128 operator~(B128 a) { return {~a.lo, ~a.hi}; }
__device__ __forceinline__ B128 operator<<(B128 a, int k) {
  return {a.lo << k, (a.hi << k) | (a.lo >> (64 - k))};
}
__device__ __forceinline__ B128 operator>>(B128 a, int k) {
  return {(a.lo >> k) | (a.hi << (64 - k)), a.hi >> k};
}
__device__ __forceinline__ bool any(B128 a) { return (a.lo | a.hi) != 0ull; }
__device__ __forceinline__ bool same(B128 a, B128 b) { return a.lo == b.lo && a.hi == b.hi; }
__device__ __forceinline__ B128 bit128(int i) {
  return i < 64 ? B128{1ull << i, 0ull} : B128{0ull, 1ull << (i - 64)};
}
__device__ __forceinline__ bool test128(B128 a, int i) {
  return ((i < 64 ? a.lo >> i : a.hi >> (i - 64)) & 1ull) != 0ull;
}

// Hex: cell xy = row * 11 + col at bit xy of a 121-bit board; b[c] holds colour c's stones.
// State words: b[0] (4 words, low first), b[1] (4 words), flags.  Flags: bit 0 the colour to move
// (step_count_ % 2), bit 1 player_order_[0] (player p plays colour p ^ bit 1), bit 2 "the last
// step ended the game", bit 3 step_count_ == 0, bit 4 step_count_ == 1 (the swap is legal).
// board_'s component ids are not kept: the terminal test flood-fills the mover's stones from
// the placed cell instead (the ids follow connectivity exactly, so both give the same answer).
struct Hex : BitboardState<9> {
  using Act = int32_t;
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = true;
  static constexpr int kPlayers = 2, kCells = 121, kActions = 122;
  static constexpr uint32_t kColor = 1u, kOrder = 2u, kOver = 4u, kFresh = 8u, kCanSwap = 16u;

  static __device__ __forceinline__ B128 board_mask() {
    return make_b128(0x1ffffffffffffffull, ~0ull);
  }
  static __device__ __forceinline__ B128 col0() {
    return make_b128(0x400801002004ull, 0x80100200400801ull);
  }
  static __device__ __forceinline__ B128 col10() {
    return make_b128(0x100200400801002ull, 0x40080100200400ull);
  }
  static __device__ __forceinline__ B128 row0() { return make_b128(0ull, 0x7ffull); }
  static __device__ __forceinline__ B128 row10() { return make_b128(0x1ffc00000000000ull, 0ull); }

  static __device__ __forceinline__ B128 get(const uint32_t* w) {
    return make_b128((uint64_t)w[2] | ((uint64_t)w[3] << 32), (uint64_t)w[0] | ((uint64_t)w[1] << 32));
  }
  static __device__ __forceinline__ void put(uint32_t* w, B128 x) {
    w[0] = (uint32_t)x.lo;
    w[1] = (uint32_t)(x.lo >> 32);
    w[2] = (uint32_t)x.hi;
    w[3] = (uint32_t)(x.hi >> 32);
  }

  // The six neighbours of (row, col): (row, col -+ 1) = -+1, (row -+ 1, col) = -+11,
  // (row + 1, col - 1) = +10, (row - 1, col + 1) = -10 (HexEnv::Neighbour).
  static __device__ __forceinline__ B128 spread(B128 r) {
    const B128 w = r & ~col0(), e = r & ~col10();
    return (r | (w >> 1) | (e << 1) | (w << 10) | (e >> 10) | (r << 11) | (r >> 11)) &
           board_mask();
  }
  // Does the mover's group through `cell` join its two edges?  Colour 0 joins rows 0 and 10,
  // colour 1 columns 0 and 10 (HexEnv::IsTerminal, which runs after the colour flips).
  static __device__ __forceinline__ bool joins(B128 mine, int cell, int color) {
    const B128 a = color ? col0() : row0(), z = color ? col10() : row10();
    if (!any(mine & a) || !any(mine & z)) return false;
    B128 g = bit128(cell);
    for (;;) {
      const B128 next = spread(g) & mine;
      if (same(next, g)) break;
      g = next;
    }
    return any(g & a) && any(g & z);
  }

  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
#pragma unroll
    for (int k = 0; k < 8; ++k) s.w[k] = 0u;
    s.w[8] = kFresh | ((rng->next() & 1u) ? kOrder : 0u);
    so.reward = 0.0f;
    so.extra = 0.0f;
  }

  // HexEnv::Step: any in-range action runs StepGame (Place or Swap), legal or not; an illegal
  // one then ends the game with IllegalRewards(the mover).
  static __device__ __forceinline__ void step(const StateView&, State& s, Act act, int, int& done,
                                              Mt*, StepOut& so) {
    uint32_t f = s.w[8];
    B128 b[2] = {get(s.w), get(s.w + 4)};
    const int color = (int)(f & kColor);
    const uint32_t mover = (f & kColor) ^ ((f & kOrder) >> 1);
    const bool in_range = act >= 0 && act <= 121;
    const B128 occ = b[0] | b[1];
    const bool illegal =
        !in_range || (act < 121 ? test128(occ, act) : (f & kCanSwap) == 0u);
    bool won = false;
    if (in_range) {
      B128 mine = color ? b[1] : b[0], theirs = color ? b[0] : b[1];
      if (act < 121) {  // Place: the cell becomes the mover's, whatever was on it
        const B128 bit = bit128(act);
        mine = mine | bit;
        theirs = theirs & ~bit;
        won = joins(mine, act, color);
      } else if (any(occ)) {  // Swap: the first stone in row-major order moves to its transpose
        const int ix = occ.lo ? __ffsll((long long)occ.lo) - 1 : 63 + __ffsll((long long)occ.hi);
        const int row = ix / 11, col = ix - row * 11, sw = col * 11 + row;
        mine = (mine & ~bit128(ix)) | bit128(sw);
        theirs = theirs & ~bit128(ix) & ~bit128(sw);
      }
      b[0] = color ? theirs : mine;
      b[1] = color ? mine : theirs;
      f ^= kColor;
      f = (f & ~(kFresh | kCanSwap)) | ((f & kFresh) ? kCanSwap : 0u);
    }
    float r_mover = 0.0f;
    if (illegal) {
      done = 1;
      r_mover = -1.0f;
    } else {
      done = won;
      r_mover = won ? 1.0f : 0.0f;
    }
    f = done ? (f | kOver) : (f & ~kOver);
    put(s.w, b[0]);
    put(s.w + 4, b[1]);
    s.w[8] = f;
    so.reward = mover ? -r_mover : r_mover;
    so.extra = -so.reward;
    if (r_mover == 0.0f) so.reward = so.extra = 0.0f;
  }

  // obs[player][row][col][plane] is one 4-byte word per (player, cell): planes 0 and 1 the
  // player's own and the opponent's stones, plane 2 "the player's colour is 1", plane 3
  // step_count_ == 1.  info:board is Sign(board_), +1 for the stones of the player to move.
  template <int kB>
  static __device__ __forceinline__ void block_write_obs(const OutView& ov, int64_t row0,
                                                         int64_t row_end, bool active,
                                                         const State& s, const StepOut&) {
    __shared__ uint64_t sb[2][2][kB];  // [colour][low, high word]
    __shared__ uint32_t sf[kB];
    if (active) {
      const int64_t row = row0 + threadIdx.x;
      sb[0][0][threadIdx.x] = (uint64_t)s.w[0] | ((uint64_t)s.w[1] << 32);
      sb[0][1][threadIdx.x] = (uint64_t)s.w[2] | ((uint64_t)s.w[3] << 32);
      sb[1][0][threadIdx.x] = (uint64_t)s.w[4] | ((uint64_t)s.w[5] << 32);
      sb[1][1][threadIdx.x] = (uint64_t)s.w[6] | ((uint64_t)s.w[7] << 32);
      const uint32_t f = s.w[8];
      sf[threadIdx.x] = f;
      if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[row] = (int32_t)((f ^ (f >> 1)) & 1u);
      if (ov.env[4]) reinterpret_cast<int2*>(ov.env[4])[row] = make_int2(0, 1);
    }
    __syncthreads();
    int64_t rows = row_end - row0;
    if (rows > kB) rows = kB;
    auto stone = [&](int c, int e, int cell) -> uint32_t {
      return (uint32_t)(sb[c][cell >> 6][e] >> (cell & 63)) & 1u;
    };
    if (ov.env[0]) {
      uint32_t* obs = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(ov.env[0]) +
                                                  row0 * (2 * kCells * 4));
      const int nw = (int)rows * (2 * kCells);
      for (int v = threadIdx.x; v < nw; v += kB) {
        const int e = v / (2 * kCells), k = v - e * (2 * kCells);
        const int p = k >= kCells, cell = k - p * kCells;
        const uint32_t f = sf[e];
        const uint32_t c = (uint32_t)p ^ ((f >> 1) & 1u);  // the player's colour
        obs[v] = stone(c, e, cell) | (stone(c ^ 1u, e, cell) << 8) | (c << 16) |
                 (((f >> 4) & 1u) << 24);
      }
    }
    if (ov.env[1]) {
      int32_t* board = static_cast<int32_t*>(ov.env[1]) + row0 * kCells;
      const int nv = (int)rows * kCells;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v / kCells, cell = v - e * kCells;
        const uint32_t c = sf[e] & kColor;
        board[v] = stone(c, e, cell) ? 1 : (stone(c ^ 1u, e, cell) ? -1 : 0);
      }
    }
    if (ov.env[3]) {
      uint8_t* mask = static_cast<uint8_t*>(ov.env[3]) + row0 * kActions;
      const int nv = (int)rows * kActions;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v / kActions, a = v - e * kActions;
        const uint32_t f = sf[e];
        const bool legal = a < kCells ? !(stone(0, e, a) | stone(1, e, a)) : (f & kCanSwap) != 0u;
        mask[v] = (f & kOver) || legal ? 1 : 0;
      }
    }
    __syncthreads();
  }
};

// Othello: cell xy = row * 8 + col at bit xy.  b[0] holds the stones of the player to move,
// b[1] the opponent's -- board_ as the reference keeps it, relative to the mover.  State words:
// b[0] lo, hi, b[1] lo, hi, flags.  Flags: bit 0 current_player_, bit 1 passed_, bit 2 "the last
// step ended the game".  The legal mask is a function of the board and is recomputed where it
// is written.
struct Othello : BitboardState<5> {
  using Act = int32_t;
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = true;
  static constexpr int kPlayers = 2, kCells = 64, kActions = 65;
  static constexpr uint32_t kPlayer = 1u, kPassed = 2u, kOver = 4u;
  static constexpr uint64_t kNotCol0 = 0xfefefefefefefefeull, kNotCol7 = 0x7f7f7f7f7f7f7f7full;

  // one step of direction d (board_games.h kOthelloShifts order: +1, -1, +8, -8, +7, -7, +9,
  // -9); a step that would wrap across column 0 or 7 leaves the board
  static __device__ __forceinline__ uint64_t shift(uint64_t x, int d) {
    switch (d) {
      case 0: return (x << 1) & kNotCol0;
      case 1: return (x >> 1) & kNotCol7;
      case 2: return x << 8;
      case 3: return x >> 8;
      case 4: return (x << 7) & kNotCol7;
      case 5: return (x >> 7) & kNotCol0;
      case 6: return (x << 9) & kNotCol0;
      default: return (x >> 9) & kNotCol7;
    }
  }
  // the empty cells from which `own` captures along some line of `other` stones
  static __device__ __forceinline__ uint64_t moves(uint64_t own, uint64_t other) {
    const uint64_t empty = ~(own | other);
    uint64_t m = 0ull;
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      uint64_t t = shift(own, d) & other;
#pragma unroll
      for (int k = 0; k < 5; ++k) t |= shift(t, d) & other;
      m |= shift(t, d) & empty;
    }
    return m;
  }
  static __device__ __forceinline__ uint64_t load_board(const uint32_t* w) {
    return (uint64_t)w[0] | ((uint64_t)w[1] << 32);
  }

  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    const uint64_t my = (1ull << 28) | (1ull << 35), opp = (1ull << 27) | (1ull << 36);
    s.w[0] = (uint32_t)my;
    s.w[1] = (uint32_t)(my >> 32);
    s.w[2] = (uint32_t)opp;
    s.w[3] = (uint32_t)(opp >> 32);
    s.w[4] = (rng->next() & 1u) ? kPlayer : 0u;
    so.reward = 0.0f;
    so.extra = 0.0f;
  }

  // OthelloEnv::Step.  An in-range action runs StepGame, legal or not: every capturing line
  // from the action cell flips (Captures does not look at the cell itself) and the cell joins
  // the mover, unless it was the opponent's -- OpponentBoardValue then keeps it theirs.
  static __device__ __forceinline__ void step(const StateView&, State& s, Act act, int, int& done,
                                              Mt*, StepOut& so) {
    uint64_t my = load_board(s.w), opp = load_board(s.w + 2);
    uint32_t f = s.w[4];
    const uint32_t mover = f & kPlayer;
    const bool in_range = act >= 0 && act <= 64;
    bool illegal = !in_range;
    if (in_range) {
      const uint64_t legal = moves(my, opp);
      illegal = act < 64 ? ((legal >> act) & 1ull) == 0ull : legal != 0ull;
    }
    float r0 = 0.0f, r1 = 0.0f;  // players 0 and 1
    bool ended = false;
    if (in_range) {
      if (act < 64) {
        const uint64_t x = 1ull << act;
        uint64_t flips = 0ull;
#pragma unroll
        for (int d = 0; d < 8; ++d) {
          uint64_t run = 0ull, cur = shift(x, d);
          while (cur & opp) {
            run |= cur;
            cur = shift(cur, d);
          }
          if (cur & my) flips |= run;
        }
        my |= flips | x;
        opp &= ~flips;
      }
      ended = (my | opp) == ~0ull || opp == 0ull || ((f & kPassed) && act == 64);
      if (ended) {  // GetReward: stone counts from the mover's side (the overlap counts twice)
        const int mc = __popcll(my), oc = __popcll(opp);
        if (mc != oc) {
          const uint32_t winner = mc > oc ? mover : mover ^ 1u;
          r0 = winner ? -1.0f : 1.0f;
          r1 = -r0;
        }
      }
      const uint64_t next_my = opp, next_opp = my & ~opp;
      my = next_my;
      opp = next_opp;
      f = (f ^ kPlayer) & ~kPassed;
      if (act == 64) f |= kPassed;
    }
    if (illegal) {
      done = 1;
      r0 = mover ? 1.0f : -1.0f;
      r1 = -r0;
    } else {
      done = ended;
    }
    f = done ? (f | kOver) : (f & ~kOver);
    s.w[0] = (uint32_t)my;
    s.w[1] = (uint32_t)(my >> 32);
    s.w[2] = (uint32_t)opp;
    s.w[3] = (uint32_t)(opp >> 32);
    s.w[4] = f;
    so.reward = r0;
    so.extra = r1;
  }

  // obs[player][row][col][plane]: plane 0 the player's own stones, plane 1 the opponent's, two
  // cells per 4-byte word.  info:board is board_ itself: +1 for the player to move.
  template <int kB>
  static __device__ __forceinline__ void block_write_obs(const OutView& ov, int64_t row0,
                                                         int64_t row_end, bool active,
                                                         const State& s, const StepOut&) {
    __shared__ uint64_t sb[3][kB];  // the mover's stones, the opponent's, the legal moves
    __shared__ uint32_t sf[kB];
    if (active) {
      const int64_t row = row0 + threadIdx.x;
      const uint64_t my = load_board(s.w), opp = load_board(s.w + 2);
      const uint32_t f = s.w[4];
      sb[0][threadIdx.x] = my;
      sb[1][threadIdx.x] = opp;
      sb[2][threadIdx.x] = ov.env[3] ? moves(my, opp) : 0ull;
      sf[threadIdx.x] = f;
      if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[row] = (int32_t)(f & kPlayer);
      if (ov.env[4]) reinterpret_cast<int2*>(ov.env[4])[row] = make_int2(0, 1);
    }
    __syncthreads();
    int64_t rows = row_end - row0;
    if (rows > kB) rows = kB;
    if (ov.env[0]) {
      constexpr int kWordsPerEnv = 2 * kCells * 2 / 4;
      uint32_t* obs = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(ov.env[0]) +
                                                  row0 * (2 * kCells * 2));
      const int nw = (int)rows * kWordsPerEnv;
      for (int v = threadIdx.x; v < nw; v += kB) {
        const int e = v / kWordsPerEnv, k = v - e * kWordsPerEnv;
        const int p = k >= kCells / 2, cell = 2 * (k - p * (kCells / 2));
        const uint32_t other = (uint32_t)p ^ (sf[e] & kPlayer);  // 1: the player is not to move
        const uint32_t own2 = (uint32_t)(sb[other][e] >> cell) & 3u;
        const uint32_t opp2 = (uint32_t)(sb[other ^ 1u][e] >> cell) & 3u;
        obs[v] = (own2 & 1u) | ((opp2 & 1u) << 8) | ((own2 >> 1) << 16) | ((opp2 >> 1) << 24);
      }
    }
    if (ov.env[1]) {
      int32_t* board = static_cast<int32_t*>(ov.env[1]) + row0 * kCells;
      const int nv = (int)rows * kCells;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v >> 6, cell = v & 63;
        board[v] = ((sb[0][e] >> cell) & 1ull) ? 1 : (((sb[1][e] >> cell) & 1ull) ? -1 : 0);
      }
    }
    if (ov.env[3]) {
      uint8_t* mask = static_cast<uint8_t*>(ov.env[3]) + row0 * kActions;
      const int nv = (int)rows * kActions;
      for (int v = threadIdx.x; v < nv; v += kB) {
        const int e = v / kActions, a = v - e * kActions;
        const uint64_t legal = sb[2][e];
        const bool m = a < kCells ? ((legal >> a) & 1ull) != 0ull : legal == 0ull;
        mask[v] = (sf[e] & kOver) || m ? 1 : 0;
      }
    }
    __syncthreads();
  }
};

// pgx/board_games.h TicTacToeEnvFns / ConnectFourEnvFns / HexEnvFns / OthelloEnvFns::StateSpec.  No options: any iopt is
// accepted and ignored, and so is the precision (no real-valued state).  Reset draws (one
// word) are not counted in bytes_per_env_step.
const KindDesc kPgxKinds[] = {
    {.kind = EPB_TIC_TAC_TOE,
     .keys = {{"obs", EPB_BOOL, 3, {3, 3, 2}, true}, {"info:board", EPB_I32, 2, {3, 3}},
              {"info:current_player", EPB_I32, 0, {}}, {"info:legal_action_mask", EPB_BOOL, 1, {9}},
              {"info:players.id", EPB_I32, 0, {}, true}},
     .action = kDiscreteAction, .NI = kStateWords<TicTacToe>, .fp64_only = true,
     .launch = fixed_launch<TicTacToe>, .players = TicTacToe::kPlayers},
    {.kind = EPB_CONNECT_FOUR,
     .keys = {{"obs", EPB_BOOL, 3, {6, 7, 2}, true}, {"info:board", EPB_I32, 2, {6, 7}},
              {"info:current_player", EPB_I32, 0, {}}, {"info:legal_action_mask", EPB_BOOL, 1, {7}},
              {"info:players.id", EPB_I32, 0, {}, true}},
     .action = kDiscreteAction, .NI = kStateWords<ConnectFour>, .fp64_only = true,
     .launch = fixed_launch<ConnectFour>, .players = ConnectFour::kPlayers},
    {.kind = EPB_HEX,
     .keys = {{"obs", EPB_BOOL, 3, {11, 11, 4}, true}, {"info:board", EPB_I32, 2, {11, 11}},
              {"info:current_player", EPB_I32, 0, {}},
              {"info:legal_action_mask", EPB_BOOL, 1, {122}},
              {"info:players.id", EPB_I32, 0, {}, true}},
     .action = kDiscreteAction, .NI = kStateWords<Hex>, .fp64_only = true,
     .launch = fixed_launch<Hex>, .players = Hex::kPlayers},
    {.kind = EPB_OTHELLO,
     .keys = {{"obs", EPB_BOOL, 3, {8, 8, 2}, true}, {"info:board", EPB_I32, 2, {8, 8}},
              {"info:current_player", EPB_I32, 0, {}},
              {"info:legal_action_mask", EPB_BOOL, 1, {65}},
              {"info:players.id", EPB_I32, 0, {}, true}},
     .action = kDiscreteAction, .NI = kStateWords<Othello>, .fp64_only = true,
     .launch = fixed_launch<Othello>, .players = Othello::kPlayers},
};
const KindDesc* pgx_kind(int kind) {
  if (const KindDesc* d = find_kind(kPgxKinds, kind)) return d;
  if (const KindDesc* d = go_kind(kind)) return d;  // Go9x9, Go13x13, Go19x19 (go.cu)
  return chess_kind(kind);                           // Chess, GardnerChess (chess.cu)
}

}  // namespace epb
