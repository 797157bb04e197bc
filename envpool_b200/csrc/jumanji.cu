// Jumanji family: Game2048-v1, bit-exact with the reference (jumanji/game2048_env.h) including
// the libstdc++ mt19937 distribution semantics of its random cell.  One CUDA thread per env.
//
// State: the 16 tile exponents (0 = empty) at 5 bits each -- cell c = row * 4 + col lives in
// word c / 6 at bit 5 * (c % 6) -- plus the action mask of the board in bits 20..23 of word 2.
// Exponents stay <= 30: configured cells are at most 26 (capi.cu), and sixteen tiles of 2^26
// merge into one tile of 2^30 at most, so 5 bits hold every reachable tile.
//
// Each step computes the four directions once, for the board it leaves behind: that gives the
// action mask (written out, and stored in the state) and `done` (no direction moves).  The next
// step reads whether its action moves the board from the stored mask instead of recomputing it.
//
// The pool's configured boards (game2048_initial_board, game2048_replay_boards) sit in the
// state blob where real-valued envs keep rstate, packed like the state: words 0..2 the initial
// board, words 3 + 3 k .. 5 + 3 k replay board k (capi.cu epb_game2048_boards).  iopt bit 0 is
// add_random_cell, bit 1 "an initial board is configured", bit 2 "replay boards are configured".
#include "common.cuh"

namespace epb {

struct Game2048 {
  using Act = int32_t;
  struct State { int32_t w0, w1, w2; };
  static constexpr bool kRngInReset = true, kRngInStep = true, kBlockObs = false;
  static constexpr bool kResetDone = true;  // a configured board may have no legal move
  static constexpr int kReplaySteps = 32;

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

launch_fn jumanji_step_fn(int kind) { return kind == 12 ? launch_step<Game2048> : nullptr; }
launch_fn jumanji_rollout_fn(int kind) {
  return kind == 12 ? launch_rollout<Game2048> : nullptr;
}

}  // namespace epb
