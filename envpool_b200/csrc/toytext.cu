// toy_text family: FrozenLake, Catch, Taxi, NChain, CliffWalking, Blackjack -- integer MDPs,
// bit-exact with the reference including the libstdc++ mt19937 distribution semantics.
// One CUDA thread per env; each env's whole integer state is packed in one or two 32-bit
// words.  Each step() cites the reference lines it restates (paths relative to
// the reference tree's envpool/toy_text/).
#include "common.cuh"

namespace epb {

struct IntState1 { int32_t w; };
struct IntState2 { int32_t w0, w1; };
__device__ __forceinline__ void load_i1(const StateView& sv, int e, IntState1& s) {
  s.w = sv.istate[e];
}
__device__ __forceinline__ void store_i1(const StateView& sv, int e, const IntState1& s) {
  sv.istate[e] = s.w;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) {
  return v < lo ? lo : (v > hi ? hi : v);
}

// --------------------------------------------------------------------------- FrozenLake
// frozen_lake.h:58-108.  Maps (frozen_lake.h:63-69) as hole/goal bit masks indexed by
// x*size+y.
//
// State word: x | y<<3 | slip-queue<<6.  The env draws one uniform_int(-1,1) per step and
// nothing at reset, so its mt19937 words are consumed strictly in order; instead of touching
// the table every step (one 32-B sector for 4 useful bytes), a whole chunk of 8 words is
// regenerated at once (4 sector reads + 1 write, common.cuh Mt::regen) and the 8 resulting
// draws are queued in the state word as 2-bit codes under a marker bit: 0..2 = Lemire result
// (uniform_int_dist.h:252-282 with range 3: product>>32), 3 = that word was REJECTED by
// Lemire's test (low < 2^32 mod 3 = 1, i.e. the word is 0) and the next word decides.  Same
// draws, same order, same results as drawing lazily -- RNG traffic drops from 32 to ~20 B per
// step and 7 of 8 steps touch no RNG memory at all.
struct FrozenLake {
  using Act = int32_t;
  using State = IntState1;
  static constexpr bool kRngInReset = false, kRngInStep = true, kBlockObs = false;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) { load_i1(sv, e, s); }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) { store_i1(sv, e, s); }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt*, StepOut& so) {
    s.w &= ~63;  // x = y = 0; the slip queue survives the episode boundary
    if ((s.w >> 6) == 0) s.w |= 1 << 6;  // empty queue = marker bit only
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ int pop_slip(uint32_t& queue, Mt* rng) {
    for (;;) {
      if (queue <= 1u) {  // empty: draw the next 8 engine words in one go
        uint32_t w[8];
        rng->next_batch<8>(w);
        queue = 1u;
#pragma unroll
        for (int k = 7; k >= 0; --k) {
          uint32_t code = w[k] == 0u ? 3u : (uint32_t)(((uint64_t)w[k] * 3ull) >> 32);
          queue = (queue << 2) | code;
        }
      }
      uint32_t code = queue & 3u;
      queue >>= 2;
      if (code != 3u) return (int)code - 1;
    }
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt* rng, StepOut& so) {
    // "SFFF","FHFH","FFFH","HFFG": holes at cells 5,7,11,12; goal 15
    const uint64_t kHole4 = (1ull << 5) | (1ull << 7) | (1ull << 11) | (1ull << 12);
    const uint64_t kGoal4 = 1ull << 15;
    // 8x8 map rows: holes at (2,3)(3,5)(4,3)(5,1)(5,2)(5,6)(6,1)(6,4)(6,6)(7,3); goal (7,7)
    const uint64_t kHole8 = (1ull << 19) | (1ull << 29) | (1ull << 35) | (1ull << 41) |
                            (1ull << 42) | (1ull << 46) | (1ull << 49) | (1ull << 52) |
                            (1ull << 54) | (1ull << 59);
    const uint64_t kGoal8 = 1ull << 63;
    const int size = sv.iopt;
    int x = s.w & 7, y = (s.w >> 3) & 7;
    uint32_t queue = (uint32_t)s.w >> 6;
    done = (cur >= sv.max_steps);
    act = (act + pop_slip(queue, rng) + 4) % 4;
    if (act == 0) {
      --y;
    } else if (act == 1) {
      ++x;
    } else if (act == 2) {
      ++y;
    } else {
      --x;
    }
    x = clampi(x, 0, size - 1);
    y = clampi(y, 0, size - 1);
    int cell = x * size + y;
    uint64_t hole = size != 8 ? kHole4 : kHole8, goal = size != 8 ? kGoal4 : kGoal8;
    float reward = 0.0f;
    if (((hole | goal) >> cell) & 1ull) {
      done = 1;
      reward = ((goal >> cell) & 1ull) ? 1.0f : 0.0f;
    }
    s.w = (int32_t)((uint32_t)x | ((uint32_t)y << 3) | (queue << 6));
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (!ov.env[0]) return;
    int x = s.w & 7, y = (s.w >> 3) & 7;
    static_cast<int32_t*>(ov.env[0])[row] = x * sv.iopt + y;
  }
};

// -------------------------------------------------------------------------------- Catch
// catch.h:62-93.  State: x | y<<8 | paddle<<16 (height 10, width 5: the registered and
// default config, toy_text/registration.py:19-27).  The 10x5 float grid is zero except the
// ball and paddle cells; the reference relies on a zero-initialised StateBuffer for that
// (state_buffer_queue.h) -- here the whole 200 B row is written, block-cooperatively so
// every store instruction covers contiguous 16 B chunks.
struct Catch {
  using Act = int32_t;
  using State = IntState1;
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = true;
  static constexpr int kH = 10, kW = 5, kCells = kH * kW;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) { load_i1(sv, e, s); }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) { store_i1(sv, e, s); }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng, StepOut& so) {
    int y = rng->uniform_int(0, kW - 1);
    s.w = 0 | (y << 8) | ((kW / 2) << 16);
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView&, State& s, Act act, int,
                                              int& done, Mt*, StepOut& so) {
    int x = s.w & 0xff, y = (s.w >> 8) & 0xff, paddle = (s.w >> 16) & 0xff;
    float reward = 0.0f;
    paddle += act - 1;
    if (paddle < 0) paddle = 0;
    if (paddle >= kW) paddle = kW - 1;
    if (++x == kH - 1) {
      done = 1;
      reward = y == paddle ? 1.0f : -1.0f;
    }
    s.w = x | (y << 8) | (paddle << 16);
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView&, const OutView&, int64_t,
                                                   const State&,
                                                   const StepOut&) {}
  // rows [row0, row0+kBlock) ∩ [.., row_end) of the obs column are written by the CTA.
  template <int kB>
  static __device__ __forceinline__ void block_write_obs(const OutView& ov, int64_t row0,
                                                         int64_t row_end, bool active,
                                                         const State& s, const StepOut&) {
    __shared__ int16_t cells[kB][2];
    int x = s.w & 0xff, y = (s.w >> 8) & 0xff, paddle = (s.w >> 16) & 0xff;
    cells[threadIdx.x][0] = active ? (int16_t)(x * kW + y) : (int16_t)-1;
    cells[threadIdx.x][1] = active ? (int16_t)((kH - 1) * kW + paddle) : (int16_t)-1;
    __syncthreads();
    if (ov.env[0]) {
      int64_t rows = row_end - row0;
      if (rows > kB) rows = kB;
      int nvec = (int)(rows * kCells / 2);  // float2 chunks (kCells is even)
      float2* out = reinterpret_cast<float2*>(static_cast<float*>(ov.env[0]) + row0 * kCells);
      for (int v = threadIdx.x; v < nvec; v += kB) {
        int e = (2 * v) / kCells;
        int c = (2 * v) - e * kCells;
        int b = cells[e][0], p = cells[e][1];
        out[v] = make_float2((c == b || c == p) ? 1.0f : 0.0f,
                             (c + 1 == b || c + 1 == p) ? 1.0f : 0.0f);
      }
    }
    __syncthreads();
  }
};

// --------------------------------------------------------------------------------- Taxi
// taxi.h:69-127.  State: x | y<<4 | s<<8 | t<<12.
struct Taxi {
  using Act = int32_t;
  using State = IntState1;
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = false;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) { load_i1(sv, e, s); }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) { store_i1(sv, e, s); }
  static __device__ __forceinline__ void reset(const StateView&, State& st, Mt* rng, StepOut& so) {
    MtIntBatch<4> b(*rng);
    int x = b.uniform_int(0, 4);
    int y = b.uniform_int(0, 4);
    int s = b.uniform_int(0, 3);
    int t = b.uniform_int(0, 3);
    st.w = x | (y << 4) | (s << 8) | (t << 12);
    so.reward = 0.0f;
  }
  // map_ rows "|:|::|","|:|::|","|::::|","||:|:|","||:|:|": bit (x*6+c) set iff map[x][c]==':'
  static __device__ __forceinline__ bool colon(int x, int c) {
    const uint32_t kColon = (0b011010u) | (0b011010u << 6) | (0b011110u << 12) |
                            (0b010100u << 18) | (0b010100u << 24);
    return (kColon >> (x * 6 + c)) & 1u;
  }
  // loc_map_ "0   1","     ","     ","     ","2  3 ": depot id at (x,y) or -1
  static __device__ __forceinline__ int depot(int x, int y) {
    if (x == 0 && y == 0) return 0;
    if (x == 0 && y == 4) return 1;
    if (x == 4 && y == 0) return 2;
    if (x == 4 && y == 3) return 3;
    return -1;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& st, Act act, int cur,
                                              int& done, Mt*, StepOut& so) {
    int x = st.w & 0xf, y = (st.w >> 4) & 0xf, s = (st.w >> 8) & 0xf, t = (st.w >> 12) & 0xf;
    done = (cur >= sv.max_steps);
    float reward = -1.0f;
    if (act == 0) {
      if (x < 4) ++x;
    } else if (act == 1) {
      if (x > 0) --x;
    } else if (act == 2) {
      if (colon(x, y + 1)) ++y;
    } else if (act == 3) {
      if (colon(x, y)) --y;
    } else if (act == 4) {
      if (s < 4 && depot(x, y) == s) {
        s = 4;
      } else {
        reward = -10.0f;
      }
    } else {
      if (s == 4 && depot(x, y) == t) {
        s = t;
        done = 1;
        reward = 20.0f;
      } else if (s == 4 && depot(x, y) >= 0) {
        s = depot(x, y);
      } else {
        reward = -10.0f;
      }
    }
    st.w = x | (y << 4) | (s << 8) | (t << 12);
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& st, const StepOut&) {
    if (!ov.env[0]) return;
    int x = st.w & 0xf, y = (st.w >> 4) & 0xf, s = (st.w >> 8) & 0xf, t = (st.w >> 12) & 0xf;
    static_cast<int32_t*>(ov.env[0])[row] = ((x * 5 + y) * 5 + s) * 4 + t;
  }
};

// ------------------------------------------------------------------------------- NChain
// nchain.h:61-92.  State: s_.
struct NChain {
  using Act = int32_t;
  using State = IntState1;
  static constexpr bool kRngInReset = false, kRngInStep = true, kBlockObs = false;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) { load_i1(sv, e, s); }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) { store_i1(sv, e, s); }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt*, StepOut& so) {
    s.w = 0;
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt* rng, StepOut& so) {
    done = (cur >= sv.max_steps);
    if (rng->uniform_real(0, 1) < 0.2) act = 1 - act;
    float reward = 0.0f;
    if (act != 0) {
      reward = 2.0f;
      s.w = 0;
    } else if (s.w < 4) {
      ++s.w;
    } else {
      reward = 10.0f;
    }
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (ov.env[0]) static_cast<int32_t*>(ov.env[0])[row] = s.w;
  }
};

// ------------------------------------------------------------------------- CliffWalking
// cliffwalking.h:64-111.  State: x | y<<8.  No elapsed-step limit of its own.
template <bool kSlippery>
struct CliffWalking {
  using Act = int32_t;
  using State = IntState1;
  static constexpr bool kRngInReset = false, kRngInStep = kSlippery, kBlockObs = false;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) { load_i1(sv, e, s); }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) { store_i1(sv, e, s); }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt*, StepOut& so) {
    s.w = 3 | (0 << 8);
    so.reward = 0.0f;
    so.extra = 1.0f;
  }
  static __device__ __forceinline__ void step(const StateView&, State& s, Act act, int,
                                              int& done, Mt* rng, StepOut& so) {
    if (kSlippery) {
      // k_offsets = {-1,0,1}[uniform_int(0,2)]  (cliffwalking.h:96-103)
      act = (act + (rng->uniform_int(0, 2) - 1) + 4) % 4;
    }
    int x = s.w & 0xff, y = (s.w >> 8) & 0xff;
    float reward = -1.0f;
    if (act == 0) {
      --x;
    } else if (act == 1) {
      ++y;
    } else if (act == 2) {
      ++x;
    } else {
      --y;
    }
    x = clampi(x, 0, 3);
    y = clampi(y, 0, 11);
    // The cliff test reads the cell index, not `x == 3`: for sm_90a, ptxas (CUDA 12.9) folds
    // `x == 3` into the predicate output of the clamp's VIMNMX.RELU, and that predicate is
    // also set for x == 0 -- steps along the top row then fell into the cliff.
    // x == 3 && 0 < y < 11  <=>  36 < 12 x + y < 47.
    const int cell = x * 12 + y;
    if (cell > 36 && cell < 47) {
      reward = -100.0f;
      x = 3;
      y = 0;
    }
    if (x == 3 && y == 11) done = 1;
    s.w = x | (y << 8);
    so.reward = reward;
    so.extra = kSlippery ? 1.0f / 3.0f : 1.0f;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut& so) {
    int x = s.w & 0xff, y = (s.w >> 8) & 0xff;
    if (ov.env[0]) static_cast<int32_t*>(ov.env[0])[row] = x * 12 + y;
    if (ov.env[1]) static_cast<float*>(ov.env[1])[row] = so.extra;
  }
};

// ---------------------------------------------------------------------------- Blackjack
// blackjack.h:65-147.  The reference keeps both hands as std::vector<int>; every quantity
// it ever derives from a hand (SumHand, UsableAce, IsNatural, dealer_[0]) is a function of
// (raw sum, has-ace, card count, first two cards), which is what is stored:
//   word = sum(6b) | ace<<6 | n<<7 (5b) | c0<<12 (4b) | c1<<16 (4b);  w0 = player, w1 = dealer
struct Blackjack {
  using Act = int32_t;
  using State = IntState2;
  static constexpr bool kRngInReset = true, kRngInStep = true, kBlockObs = false;
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    s.w0 = sv.istate[e];
    s.w1 = sv.istate[(int64_t)sv.n_envs + e];
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    sv.istate[e] = s.w0;
    sv.istate[(int64_t)sv.n_envs + e] = s.w1;
  }
  struct Hand {
    int sum, ace, n, c0, c1;
    __device__ __forceinline__ explicit Hand(int w)
        : sum(w & 63), ace((w >> 6) & 1), n((w >> 7) & 31), c0((w >> 12) & 15),
          c1((w >> 16) & 15) {}
    __device__ __forceinline__ Hand() : sum(0), ace(0), n(0), c0(0), c1(0) {}
    __device__ __forceinline__ int pack() const {
      return sum | (ace << 6) | (n << 7) | (c0 << 12) | (c1 << 16);
    }
    __device__ __forceinline__ void push(int c) {  // player_.push_back(DrawCard())
      if (n == 0) c0 = c;
      if (n == 1) c1 = c;
      sum += c;
      ace |= (c == 1);
      if (n < 31) ++n;
    }
    // SumHand / UsableAce / Score / IsNatural: blackjack.h:110-146
    __device__ __forceinline__ int sum_hand() const {
      return (ace && sum + 10 <= 21) ? sum + 10 : sum;
    }
    __device__ __forceinline__ int score() const {
      int r = sum_hand();
      return r > 21 ? 0 : r;
    }
    __device__ __forceinline__ bool natural() const {
      return n == 2 && ((c0 == 1 && c1 == 10) || (c0 == 10 && c1 == 1));
    }
  };
  template <class Rng>
  static __device__ __forceinline__ int draw(Rng* rng) {  // DrawCard, blackjack.h:108
    int c = rng->uniform_int(1, 13);
    return c < 10 ? c : 10;
  }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng, StepOut& so) {
    Hand p, d;
    MtIntBatch<4> b(*rng);
    p.push(draw(&b));
    p.push(draw(&b));
    d.push(draw(&b));
    d.push(draw(&b));
    s.w0 = p.pack();
    s.w1 = d.pack();
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int,
                                              int& done, Mt* rng, StepOut& so) {
    const bool natural = sv.iopt & 1, sab = (sv.iopt >> 1) & 1;
    Hand p(s.w0), d(s.w1);
    float reward = 0.0f;
    if (act != 0) {
      p.push(draw(rng));
      if (p.sum_hand() > 21) {
        done = 1;
        reward = -1.0f;
      }
    } else {
      done = 1;
      while (d.sum_hand() < 17) d.push(draw(rng));
      int ps = p.score(), ds = d.score();
      reward = (ps > ds ? 1.0f : 0.0f) - (ps < ds ? 1.0f : 0.0f);
      if (sab && p.natural() && !d.natural()) {
        reward = 1.0f;
      } else if (!sab && natural && p.natural() && reward == 1.0f) {
        reward = 1.5f;
      }
    }
    s.w0 = p.pack();
    s.w1 = d.pack();
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (!ov.env[0]) return;
    Hand p(s.w0), d(s.w1);
    int32_t* o = static_cast<int32_t*>(ov.env[0]) + row * 3;
    o[0] = p.sum_hand();
    o[1] = d.c0;
    o[2] = p.ace;
  }
};

// Per-step RNG traffic (mt19937 table and index) of the envs that draw while stepping.
constexpr int kSlipBytes = 16 + 8;  // FrozenLake, slippery CliffWalking: one uniform_int
constexpr int kNChainBytes = 32 + 8;  // one uniform_real

KindLaunch cliffwalking_launch(int, int iopt) {  // iopt: is_slippery
  return iopt ? kind_launch<CliffWalking<true>>(kSlipBytes) : kind_launch<CliffWalking<false>>();
}

// The real-state column of these pools is sized by precision although NR = 0: the state
// snapshot format keeps it.
const KindDesc kToyTextKinds[] = {
    {.kind = EPB_FROZEN_LAKE, .keys = {{"obs", EPB_I32, 0, {}}}, .action = kDiscreteAction,
     .NI = kStateWords<FrozenLake>, .default_iopt = 4, .iopts = {4, 8}, .n_iopts = 2,
     .iopt_error = "FrozenLake size must be 4 or 8",
     .launch = fixed_launch<FrozenLake, kSlipBytes>},
    {.kind = EPB_CATCH, .keys = {{"obs", EPB_F32, 2, {Catch::kH, Catch::kW}}},
     .action = kDiscreteAction, .NI = kStateWords<Catch>, .launch = fixed_launch<Catch>},
    {.kind = EPB_TAXI, .keys = {{"obs", EPB_I32, 0, {}}}, .action = kDiscreteAction,
     .NI = kStateWords<Taxi>, .launch = fixed_launch<Taxi>},
    {.kind = EPB_NCHAIN, .keys = {{"obs", EPB_I32, 0, {}}}, .action = kDiscreteAction,
     .NI = kStateWords<NChain>, .launch = fixed_launch<NChain, kNChainBytes>},
    {.kind = EPB_CLIFF_WALKING, .keys = {{"obs", EPB_I32, 0, {}}, {"info:prob", EPB_F32, 0, {}}},
     .action = kDiscreteAction, .NI = kStateWords<CliffWalking<false>>,
     .launch = cliffwalking_launch},
    // iopt: natural | sab << 1
    {.kind = EPB_BLACKJACK, .keys = {{"obs", EPB_I32, 1, {3}}}, .action = kDiscreteAction,
     .NI = kStateWords<Blackjack>, .default_iopt = 2, .launch = fixed_launch<Blackjack>},
};
const KindDesc* toytext_kind(int kind) { return find_kind(kToyTextKinds, kind); }

}  // namespace epb
