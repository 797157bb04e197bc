// PGX family: TicTacToe-v1 and ConnectFour-v1 (pgx/board_games.h TicTacToeEnv, ConnectFourEnv),
// bit-exact with the reference.  The engine's first two-player kinds: every env row has two
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
// 8 info:players.id); ConnectFour 445 = 4 + 2 x (4 + 20) + 38 + 355 (168, 168, 4, 7, 8).
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

// pgx/board_games.h TicTacToeEnvFns / ConnectFourEnvFns::StateSpec.  No options: any iopt is
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
};
const KindDesc* pgx_kind(int kind) { return find_kind(kPgxKinds, kind); }

}  // namespace epb
