// envpool_b200 device-side core: SoA pool views, the device std::mt19937 + libstdc++
// distribution recipes, and the generic thread-per-env step / rollout kernels that every
// classic_control and toy_text env plugs into.
//
// What this replaces in the reference (paths relative to the reference tree's envpool/):
//   core/async_envpool.h:59-82   Send: batch action -> per-env ActionSlice   (action gather)
//   core/async_envpool.h:118-131 worker loop: auto-reset decision + EnvStep
//   core/env.h:184-256           EnvStep / PreProcess / Allocate (common columns)
//   core/state_buffer.h:81-131   row reservation + completion counting         (obs scatter)
// On the GPU all of it is one kernel: row i of the batch is one thread, the env's state is
// a column of SoA arrays in HBM, outputs are written straight into the packed output slab.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "exchange.cuh"

namespace epb {

constexpr int kMtN = 624;
constexpr int kMtM = 397;
constexpr int kBlock = 128;  // threads per CTA for thread-per-env kernels

// Persistent per-env state, structure-of-arrays over the local env index.
struct StateView {
  int32_t n_envs;         // N: SoA stride (envs owned by this pool)
  int32_t max_steps;      // config max_episode_steps (INT_MAX when unset)
  int32_t env_id_offset;  // global id of local env 0
  int32_t iopt;           // env option (size / version / is_slippery / natural|sab<<1)
  int32_t* flags;         // (current_step_ << 1) | done_      (env.h:81, cartpole.h:67)
  uint32_t* mt;           // [624][N] mt19937 words
  int32_t* mt_idx;        // [N] index of the next word to regenerate, 0..623
  void* rstate;           // [NR][N] real state (double or float)
  int32_t* istate;        // [NI][N] integer state
  // Reset-ahead records (envs whose Reset() is a pure function of their RNG stream:
  // classic_control).  Every env owns a ring of rec_q records = its NEXT rec_q initial states,
  // drawn ahead of time by refill_kernel, so the step kernel's auto-reset is a 32-byte load
  // instead of a dependent mt19937 round trip on one lane of the warp.  Records are produced
  // and consumed in order and these envs draw only at reset, so every trajectory stays the one
  // std::mt19937(seed + env_id) gives.  rcons / rprod count consumed / produced records
  // (mod 256; valid = rprod - rcons <= rec_q); slot of record i is i % rec_q.
  void* rec;              // [N][rec_q][NR] real: one or two 16-byte loads per record
  uint8_t* rcons;         // [N] records consumed so far (written by the step kernels)
  uint8_t* rprod;         // [N] records produced so far (written by refill_kernel)
  int32_t rec_q;          // ring size, a power of two <= 16
};

// Output columns for one batch (pointers into a packed slab or caller arrays).
// Order = the reference's state-key order (env_spec.h:37-43), then env keys.
struct OutView {
  int32_t* env_id;       // info:env_id
  int32_t* players_id;   // info:players.env_id
  int32_t* elapsed;      // elapsed_step
  uint8_t* done;         // done
  float* reward;         // reward
  float* discount;       // discount
  int32_t* step_type;    // step_type
  uint8_t* trunc;        // trunc
  void* env[5];          // env-specific keys in declaration order
  int32_t* wire;         // sharded pools: packed common columns for the peers (exchange.cuh)
  int64_t t_stride_rows; // rollout: rows between consecutive time steps (= N)
};

// ---------------------------------------------------------------------------------------
// std::mt19937 on the device.
//
// Layout: the 624-word table of env e is cut into 78 chunks of 8 words; chunk c of env e is
// the 32-byte sector at word offset (c*N + e)*8.  One DRAM sector therefore holds 8
// consecutive words of ONE env (envs draw at different times, so a warp's lanes sit at
// different positions of their tables; with a word-major layout every 4-byte access would
// cost a whole sector), while lanes that do move in lockstep still touch adjacent sectors.
//
// Regeneration: the textbook "twist" regenerates all 624 words at once; here a chunk of 8 is
// regenerated when the read position enters it.  Word i needs the current words i, i+1 and
// i+397; inside a chunk-sized batch none of those has been regenerated earlier in the batch
// except i+1's predecessor, whose *old* value is what the recurrence wants, so the batch is
// 4 sector reads (own chunk, first word of the next, the two chunks holding i+397..i+404)
// + 1 sector write per 8 draws, all loads in flight together.  The sequence is identical to
// std::mt19937's.
struct Mt {
  uint32_t* base;   // &mt[eid*8]: word 0 of chunk 0 of this env
  int64_t cstride;  // words between consecutive chunks of one env (= 8*N)
  int idx;          // next word to hand out, 0..623
  uint32_t cw[8];   // register copy of the chunk idx lies in (raw words)
  bool have;
  // split-phase first access (begin / next): loads issued early, consumed by the first draw
  uint4 p_o0, p_o1, p_m0, p_m1;
  uint32_t p_nx, p_m2;
  int pending;  // 0 = nothing in flight, 1 = regeneration inputs, 2 = the current chunk
  __device__ __forceinline__ Mt(const StateView& sv, int eid)
      : base(sv.mt + (int64_t)eid * 8), cstride((int64_t)sv.n_envs * 8), idx(sv.mt_idx[eid]),
        have(false), pending(0) {}
  // idx already loaded by the caller (issued together with the env-state loads so the
  // draw does not pay a second dependent round trip)
  __device__ __forceinline__ Mt(const StateView& sv, int eid, int idx_)
      : base(sv.mt + (int64_t)eid * 8), cstride((int64_t)sv.n_envs * 8), idx(idx_),
        have(false), pending(0) {}
  __device__ __forceinline__ void save(const StateView& sv, int e) { sv.mt_idx[e] = idx; }

  __device__ __forceinline__ uint4* sector(int chunk) const {
    return reinterpret_cast<uint4*>(base + chunk * cstride);
  }
  static __device__ __forceinline__ uint32_t twist(uint32_t a, uint32_t b, uint32_t m) {
    uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return m ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
  }
  static __device__ __forceinline__ uint32_t temper(uint32_t v) {
    v ^= (v >> 11);
    v ^= (v << 7) & 0x9d2c5680u;
    v ^= (v << 15) & 0xefc60000u;
    v ^= (v >> 18);
    return v;
  }
  // Issue the loads the next draw will need and return without waiting for them: the
  // caller runs unrelated work (the step arithmetic of the warp's non-resetting lanes)
  // before the first draw, which then finds its operands already in registers.
  __device__ __forceinline__ void begin() {
    const int c = idx >> 3;
    if ((idx & 7) == 0) {
      load_regen_inputs(c);
      pending = 1;
    } else {
      const uint4* own = sector(c);
      p_o0 = own[0];
      p_o1 = own[1];
      pending = 2;
    }
  }
  __device__ __forceinline__ void load_regen_inputs(int c) {
    int c1 = c + 1, c49 = c + 49, c50 = c + 50;
    c1 = c1 >= 78 ? c1 - 78 : c1;
    c49 = c49 >= 78 ? c49 - 78 : c49;
    c50 = c50 >= 78 ? c50 - 78 : c50;
    const uint4* own = sector(c);
    const uint4* s50 = sector(c50);
    p_o0 = own[0];
    p_o1 = own[1];
    p_nx = reinterpret_cast<const uint32_t*>(sector(c1))[0];
    p_m0 = sector(c49)[1];                              // words 4..7 of chunk c+49
    p_m1 = s50[0];                                      // words 0..3 of chunk c+50
    p_m2 = reinterpret_cast<const uint32_t*>(s50)[4];   // word 4
  }
  // Make cw the raw words of the chunk idx lies in: regenerate it if idx enters it now,
  // else (first access of this kernel) read it back.  The ONE place the table is touched.
  __device__ __forceinline__ void enter_chunk() {
    const int c = idx >> 3;
    if ((idx & 7) == 0) {
      if (pending != 1) load_regen_inputs(c);
      pending = 0;
      const uint4 o0 = p_o0, o1 = p_o1, m0 = p_m0, m1 = p_m1;
      // word i+397 for i = 8c+k, k = 0..7: chunk c+49 words 5,6,7 then chunk c+50 words 0..4
      cw[0] = twist(o0.x, o0.y, m0.y);
      cw[1] = twist(o0.y, o0.z, m0.z);
      cw[2] = twist(o0.z, o0.w, m0.w);
      cw[3] = twist(o0.w, o1.x, m1.x);
      cw[4] = twist(o1.x, o1.y, m1.y);
      cw[5] = twist(o1.y, o1.z, m1.z);
      cw[6] = twist(o1.z, o1.w, m1.w);
      cw[7] = twist(o1.w, p_nx, p_m2);
      uint4* own = sector(c);
      own[0] = make_uint4(cw[0], cw[1], cw[2], cw[3]);
      own[1] = make_uint4(cw[4], cw[5], cw[6], cw[7]);
      have = true;
      // The NEXT regeneration (chunk c+1) will read sectors c+1 and c+50 -- both touched
      // just now, so they sit in L2 -- and c+2, c+51, which are not.  Ask L2 for those two
      // now (fire-and-forget): draws are rare events per env (a reset every ~20 steps, a slip
      // refill every 8), so by the time they are needed they are an L2 hit, not a DRAM
      // round trip on the critical path of that step's kernel.
      int c2 = c + 2, c51 = c + 51;
      c2 = c2 >= 78 ? c2 - 78 : c2;
      c51 = c51 >= 78 ? c51 - 78 : c51;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(sector(c2)));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(sector(c51)));
    } else if (!have) {
      if (pending != 2) {
        const uint4* own = sector(c);
        p_o0 = own[0];
        p_o1 = own[1];
      }
      pending = 0;
      cw[0] = p_o0.x; cw[1] = p_o0.y; cw[2] = p_o0.z; cw[3] = p_o0.w;
      cw[4] = p_o1.x; cw[5] = p_o1.y; cw[6] = p_o1.z; cw[7] = p_o1.w;
      have = true;
    }
  }
  __device__ __forceinline__ void advance(int k) {
    idx += k;
    idx = idx >= kMtN ? idx - kMtN : idx;
  }
  // K consecutive draws (the sequence K calls of std::mt19937::operator() would give).
  // Fast path: K is a power of two <= 8 and the read position is K-aligned -- true for every
  // env that always draws in groups of K (CartPole/Acrobot 8, Pendulum 4, MountainCar 2,
  // per-step single draws) -- so the K words sit in one chunk at cw[k..k+K).  Otherwise
  // word by word, in a rolled loop (rare: Blackjack's dealer, HalfCheetah's 18+ draws).
  template <int K>
  __device__ __forceinline__ void next_batch(uint32_t (&out)[K]) {
    const int k = idx & 7;
    if ((K == 1 || K == 2 || K == 4 || K == 8) && (k & (K - 1)) == 0) {
      enter_chunk();
#pragma unroll
      for (int j = 0; j < K; ++j) {
        uint32_t v = cw[j];
#pragma unroll
        for (int b = K; b < 8; b += K) v = (k == b) ? cw[b + j] : v;
        out[j] = temper(v);
      }
      advance(K);
    } else {
#pragma unroll 1
      for (int j = 0; j < K; ++j) {
        uint32_t w[1];
        next_batch<1>(w);
        out[j] = w[0];
      }
    }
  }
  __device__ __forceinline__ uint32_t next() {
    uint32_t w[1];
    next_batch<1>(w);
    return w[0];
  }

  // std::generate_canonical<double,53> (libstdc++ 13 bits/random.tcc:3349-3381) from two
  // engine outputs.  Explicit _rn intrinsics: never contracted into an FMA, whatever the
  // TU's flags.
  static __device__ __forceinline__ double canonical_from(uint32_t d1, uint32_t d2) {
    double sum = __dadd_rn((double)d1, __dmul_rn((double)d2, 4294967296.0));
    double ret = __dmul_rn(sum, 5.421010862427522170037e-20);  // exact: / 2^64
    if (ret >= 1.0) ret = 0.99999999999999988897769753748;     // nextafter(1,0)
    return ret;
  }
  __device__ __forceinline__ double canonical() {
    uint32_t d[2];
    next_batch<2>(d);
    return canonical_from(d[0], d[1]);
  }
  // std::uniform_real_distribution<double>(a,b)
  __device__ __forceinline__ double uniform_real(double a, double b) {
    return __dadd_rn(__dmul_rn(canonical(), __dsub_rn(b, a)), a);
  }
  // NC consecutive uniform_real(a,b) draws, one memory round trip
  template <int NC>
  __device__ __forceinline__ void uniform_real_batch(double a, double b, double (&out)[NC]) {
    uint32_t d[2 * NC];
    next_batch<2 * NC>(d);
#pragma unroll
    for (int k = 0; k < NC; ++k)
      out[k] = __dadd_rn(__dmul_rn(canonical_from(d[2 * k], d[2 * k + 1]), __dsub_rn(b, a)), a);
  }
  // std::uniform_int_distribution<int>(a,b): Lemire (bits/uniform_int_dist.h:252-282)
  __device__ __forceinline__ int uniform_int(int a, int b) {
    uint32_t range = (uint32_t)b - (uint32_t)a + 1u;
    uint64_t product = (uint64_t)next() * (uint64_t)range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
      uint32_t threshold = (0u - range) % range;
      while (low < threshold) {
        product = (uint64_t)next() * (uint64_t)range;
        low = (uint32_t)product;
      }
    }
    return a + (int)(product >> 32);
  }
};

// K uniform_int draws with the engine words fetched in one round trip.  Lemire's method
// almost never rejects (probability range/2^32 per draw); when it does, the extra words
// come from sequential next() calls after the batch, so the word order is unchanged.
template <int K>
struct MtIntBatch {
  Mt& rng;
  uint32_t words[K];
  int cursor;
  __device__ __forceinline__ explicit MtIntBatch(Mt& r) : rng(r), cursor(0) {
    rng.template next_batch<K>(words);
  }
  __device__ __forceinline__ uint32_t word() {
    uint32_t v = 0;
    bool hit = false;
#pragma unroll
    for (int k = 0; k < K; ++k)
      if (k == cursor) {
        v = words[k];
        hit = true;
      }
    ++cursor;
    return hit ? v : rng.next();
  }
  __device__ __forceinline__ int uniform_int(int a, int b) {
    uint32_t range = (uint32_t)b - (uint32_t)a + 1u;
    uint64_t product = (uint64_t)word() * (uint64_t)range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
      uint32_t threshold = (0u - range) % range;
      while (low < threshold) {
        product = (uint64_t)word() * (uint64_t)range;
        low = (uint32_t)product;
      }
    }
    return a + (int)(product >> 32);
  }
};

// Seeds every env's table: std::mt19937(seed) == init_genrand (env.h:113).  One thread per
// env; each of the 624 steps is a coalesced row write.
__global__ void seed_kernel(StateView sv, int base_seed, const int32_t* env_seed);

// ---------------------------------------------------------------------------------------
// Common output columns: Env::Allocate, core/env.h:224-256.
__device__ __forceinline__ void write_common(const OutView& ov, int64_t row, int global_eid,
                                             int cur, int done, float reward,
                                             int max_steps) {
  int step_type = (cur == 0) ? 0 : (done ? 2 : 1);
  if (ov.env_id) ov.env_id[row] = global_eid;
  if (ov.players_id) ov.players_id[row] = global_eid;
  if (ov.elapsed) ov.elapsed[row] = cur;
  if (ov.done) ov.done[row] = (uint8_t)done;
  if (ov.reward) ov.reward[row] = reward;
  if (ov.discount) ov.discount[row] = done ? 0.0f : 1.0f;
  if (ov.step_type) ov.step_type[row] = step_type;
  const int trunc = done && (cur >= max_steps);
  if (ov.trunc) ov.trunc[row] = (uint8_t)trunc;
  if (ov.wire) ov.wire[row] = pack_wire(cur, done, trunc);
}

// Per-env result of one EnvStep, kept in registers until the output write.
struct StepOut {
  float reward;
  float extra;  // env-specific scalar (CliffWalking info:prob)
};

// The Env concept every family member implements:
//   using Act = <action scalar type>;  struct State {...};
//   static void load(const StateView&, int eid, State&);
//   static void store(const StateView&, int eid, const State&);
//   static void reset(const StateView&, State&, Mt*, StepOut&);            // XxxEnv::Reset
//   static void step(const StateView&, State&, Act, int cur, int& done, Mt*, StepOut&);
//   static void write_obs(const StateView&, const OutView&, int64_t row, const State&,
//                         const StepOut&);
//   static constexpr bool kRngInReset, kRngInStep;  (Mt* is NULL when false)
//   static constexpr bool kBlockObs;                (block-cooperative obs write)
//
// Envs with `static constexpr bool kRecReset = true` use the reset-ahead records.
template <class Env, class = void>
struct UsesRec { static constexpr bool value = false; };
template <class Env>
struct UsesRec<Env, typename std::enable_if<Env::kRecReset>::type> {
  static constexpr bool value = true;
};

// One EnvStep (env.h:184-222) incl. the auto-reset decision (async_envpool.h:127).
//
// Reset, record envs: the state becomes the env's next record (slot rcons % rec_q) and the
// consume counter moves on; refill_kernel redraws consumed slots off the critical path.  The
// ring can never run dry: a step that resets is never `done`, so an env consumes at most one
// record every two steps, and the engine refills at least every rec_q - 2 launches (capi.cu).
// Reset, other envs: the draws happen here (Mt, chunked table).
template <class Env>
__device__ __forceinline__ void env_step(const StateView& sv, int eid, int& flags,
                                         typename Env::State& s, typename Env::Act a,
                                         bool force_reset, StepOut& so, int& mt_idx,
                                         int rcons) {
  int done = flags & 1;
  int cur = flags >> 1;
  const bool reset = force_reset || done;
  if constexpr (UsesRec<Env>::value) {
    // Branch-free over `reset`: every lane runs the step arithmetic on the state it loaded
    // (a warp almost always holds stepping lanes, so the resetting lanes ride along for
    // free; a done env's stale state is finite, the result is discarded) and the resetting
    // lanes then take their record.  With a branch, ptxas sinks the state loads into the
    // step side -- behind the arrival of `flags`, one more dependent L2 round trip.
    typename Env::State rec;
    if (reset) {
      // issued NOW, ahead of the step arithmetic that hides its latency
      Env::load_rec(sv, eid, rcons & (sv.rec_q - 1), rec);
      sv.rcons[eid] = (uint8_t)(rcons + 1);
      // ... and ask L2 for the record AFTER this one (fire and forget): the env's next reset is
      // >= 2 and typically ~20 steps away, so whatever has streamed through L2 since the ring
      // was written, that reset finds its 32 bytes on chip.  One request per resetting lane.
      Env::prefetch_rec(sv, eid, (rcons + 1) & (sv.rec_q - 1));
    }
    typename Env::State s1 = s;
    StepOut so1 = so;
    int cur1 = cur + 1, done1 = 0;
    Env::step(sv, s1, a, cur1, done1, nullptr, so1);
    s = reset ? rec : s1;
    so.reward = reset ? 0.0f : so1.reward;
    so.extra = reset ? 0.0f : so1.extra;
    cur = reset ? 0 : cur1;
    done = reset ? 0 : done1;
  } else {
    // A warp usually holds both resetting and stepping lanes.  Order of work: resetting
    // lanes ISSUE their mt19937 loads, then the stepping lanes run their arithmetic, then
    // the resetting lanes consume the loads -- the memory latency of a reset hides behind
    // the step math instead of adding to it.
    Mt rng(sv, eid, mt_idx);
    if (Env::kRngInReset && reset) rng.begin();
    if (!reset) {
      ++cur;
      Env::step(sv, s, a, cur, done, Env::kRngInStep ? &rng : nullptr, so);
    } else {
      cur = 0;
      done = 0;
      Env::reset(sv, s, Env::kRngInReset ? &rng : nullptr, so);
    }
    if (Env::kRngInReset || Env::kRngInStep) mt_idx = rng.idx;
  }
  flags = (cur << 1) | done;
}

// Compiler fence for one register value: every use of `v` is scheduled after this point.
// Used to keep the first USE of the (cold, DRAM-resident) action behind the ISSUE of the
// state loads -- ptxas otherwise hoists `act == 1` right behind the action load, and the
// in-order warp then sits out a full DRAM round trip before it even requests its state
// (measured with ncu stall sampling: 8 % of all samples on that one compare).
__device__ __forceinline__ void pin_value(int32_t& v) { asm volatile("" : "+r"(v)); }
__device__ __forceinline__ void pin_value(float& v) { asm volatile("" : "+f"(v)); }
__device__ __forceinline__ void pin_value(double& v) { asm volatile("" : "+d"(v)); }

// Single sync step of a batch: thread `row` handles env env_ids[row] (identity if NULL).
template <class Env, int kB = kBlock>
__global__ void __launch_bounds__(kB)
step_kernel(StateView sv, OutView ov, const typename Env::Act* __restrict__ action,
            const int32_t* __restrict__ env_ids, int n, int force_reset,
            const PeerView* __restrict__ peers,
            const typename Env::Act* __restrict__ next_action) {
  int row = blockIdx.x * kB + threadIdx.x;
  bool active = row < n;
  typename Env::State s;
  StepOut so;
  so.reward = 0.f;
  so.extra = 0.f;
  int eid = 0, flags = 0;
  typename Env::Act a = typename Env::Act();
  // Programmatic dependent launch: let the next step's grid start launching now, and wait
  // here for the previous kernel of the stream.  Every global load sits BEHIND the wait:
  // the action / env_ids of the device-resident path are usually written by the kernel just
  // before this one (a policy's argmax), and state and slab belong to the previous step.
  // Both instructions are no-ops when the kernel is launched without the PDL attribute.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (active) {
    constexpr bool kRng = Env::kRngInReset || Env::kRngInStep;
    constexpr bool kRec = UsesRec<Env>::value;
    eid = env_ids ? env_ids[row] : row;
    if (!force_reset) a = action[row];
    flags = sv.flags[eid];
    int mt_idx = 0, rcons = 0;
    if constexpr (kRec) {
      rcons = sv.rcons[eid];  // rides with the state loads: the record's slot is known at once
    } else if (kRng) {
      mt_idx = sv.mt_idx[eid];
    }
    const int mt_idx0 = mt_idx;
    Env::load(sv, eid, s);
    // Step chains know the action row of the NEXT step: ask L2 for it now (one 128-byte line
    // per warp, fire and forget).  The row is still read from HBM exactly once; what moves
    // off the next kernel's critical path is the DRAM latency of its only cold input -- a
    // policy that has just written the actions leaves them in L2 in the same way.
    if (next_action && (threadIdx.x & 31) == 0)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(next_action + row));
    pin_value(a);
    env_step<Env>(sv, eid, flags, s, a, force_reset != 0, so, mt_idx, rcons);
    Env::store(sv, eid, s);
    sv.flags[eid] = flags;
    if (!kRec && kRng && mt_idx != mt_idx0) sv.mt_idx[eid] = mt_idx;
    write_common(ov, row, eid + sv.env_id_offset, flags >> 1, flags & 1, so.reward,
                 sv.max_steps);
  }
  if constexpr (Env::kBlockObs) {
    Env::template block_write_obs<kB>(ov, (int64_t)blockIdx.x * kB, n, active, s, so);
  } else if (active) {
    Env::write_obs(sv, ov, row, s, so);
  }
  // sharded pools: forward this CTA's output rows to every peer GPU (exchange.cuh)
  if (peers) peer_forward_rows<kB>(peers, (int64_t)blockIdx.x * kB, n);
}

// Refills every env's record ring to rec_q valid records (draws rec_q - (rprod - rcons) new
// initial states, in order).  Runs BEHIND the steps that consumed and, in the engine's captured
// step chains, beside the following steps (a parallel graph branch).  The only kernel that
// touches the mt19937 tables of record envs.  Reading a stale rcons (a concurrent step has
// just consumed) only makes it refill one record fewer; the slots it writes are never the
// ones a concurrent step reads (those lie in [rcons, rprod), these in [rprod, rcons + rec_q)).
template <class Env>
__global__ void __launch_bounds__(kBlock) refill_kernel(StateView sv) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e >= sv.n_envs) return;
  const int q = sv.rec_q;
  const int c = sv.rcons[e];
  int p = sv.rprod[e];
  const int need = q - ((p - c) & 255);
  if (need <= 0) return;
  Mt rng(sv, e);
#pragma unroll 1
  for (int i = 0; i < need; ++i) {
    typename Env::State s;
    StepOut so;
    Env::reset(sv, s, &rng, so);
    Env::store_rec(sv, e, p & (q - 1), s);
    ++p;
  }
  rng.save(sv, e);
  sv.rprod[e] = (uint8_t)p;
}

// Fused rollout: T sync steps of all N envs in one launch; state stays in registers, the
// action stream [T,N] is read and the outputs [T,N,...] written once each.  Record envs:
// resets take the env's ring records first (the earlier draws), then draw in place, and the
// ring is refilled before the kernel ends -- the draw order per env is the sequential one.
template <class Env>
__global__ void __launch_bounds__(kBlock)
rollout_kernel(StateView sv, OutView ov, const typename Env::Act* __restrict__ actions,
               int T) {
  int eid = blockIdx.x * kBlock + threadIdx.x;
  const int n = sv.n_envs;
  bool active = eid < n;
  typename Env::State s;
  int flags = 0, mt_idx = 0;
  constexpr bool kRng = Env::kRngInReset || Env::kRngInStep;
  constexpr bool kRec = UsesRec<Env>::value;
  int rc = 0, rp = 0;  // record ring counters (consumed / produced)
  if (active) {
    flags = sv.flags[eid];
    if (kRng) mt_idx = sv.mt_idx[eid];
    Env::load(sv, eid, s);
    if constexpr (kRec) {
      rc = sv.rcons[eid];
      rp = sv.rprod[eid];
    }
  }
  typename Env::Act a_next = typename Env::Act();
  if (active && T > 0) a_next = actions[eid];
  for (int t = 0; t < T; ++t) {
    StepOut so;
    so.reward = 0.f;
    so.extra = 0.f;
    int64_t row = (int64_t)t * ov.t_stride_rows + eid;
    typename Env::Act a = a_next;
    if (active && t + 1 < T) a_next = actions[(int64_t)(t + 1) * n + eid];  // prefetch
    if (active) {
      if constexpr (kRec) {
        int done = flags & 1, cur = flags >> 1;
        if (!done) {
          ++cur;
          Env::step(sv, s, a, cur, done, nullptr, so);
        } else {
          cur = 0;
          done = 0;
          if (((rp - rc) & 255) != 0) {  // the ring first: its records are the earlier draws
            Env::load_rec(sv, eid, rc & (sv.rec_q - 1), s);
            so.reward = 0.0f;
            ++rc;
          } else {
            Mt rng(sv, eid, mt_idx);
            Env::reset(sv, s, &rng, so);
            mt_idx = rng.idx;
            // a record produced and consumed at once: the counters keep counting records, so
            // the refill below puts record i in slot i % rec_q, as the state layout promises
            ++rp;
            ++rc;
          }
        }
        flags = (cur << 1) | done;
      } else {
        env_step<Env>(sv, eid, flags, s, a, false, so, mt_idx, 0);
      }
      write_common(ov, row, eid + sv.env_id_offset, flags >> 1, flags & 1, so.reward,
                   sv.max_steps);
    }
    if constexpr (Env::kBlockObs) {
      Env::template block_write_obs<kBlock>(
          ov, (int64_t)t * ov.t_stride_rows + (int64_t)blockIdx.x * kBlock,
          (int64_t)t * ov.t_stride_rows + n, active, s, so);
    } else if (active) {
      Env::write_obs(sv, ov, row, s, so);
    }
  }
  if (active) {
    Env::store(sv, eid, s);
    sv.flags[eid] = flags;
    if constexpr (kRec) {
      const int q = sv.rec_q;
      const int need = q - ((rp - rc) & 255);
      if (need > 0) {  // leave the ring full, like refill_kernel
        Mt rng(sv, eid, mt_idx);
#pragma unroll 1
        for (int i = 0; i < need; ++i) {
          typename Env::State r;
          StepOut so;
          Env::reset(sv, r, &rng, so);
          Env::store_rec(sv, eid, rp & (q - 1), r);
          ++rp;
        }
        mt_idx = rng.idx;
      }
      sv.rcons[eid] = (uint8_t)rc;
      sv.rprod[eid] = (uint8_t)rp;
    }
    if (kRng) sv.mt_idx[eid] = mt_idx;
  }
}

// Host-side launch table filled by each family's translation unit.
struct LaunchArgs {
  StateView sv;
  OutView ov;
  const void* action;
  const int32_t* env_ids;
  int n;
  int force_reset;
  int T;  // rollout only
  cudaStream_t stream;
  const PeerView* peers;  // device pointer; non-NULL = fused peer exchange epilogue
  const void* next_action;  // step chains: action row of the following step (L2 prefetch)
};
typedef cudaError_t (*launch_fn)(const LaunchArgs&);

// ENVPOOL_B200_PDL=0 turns the programmatic-dependent-launch attribute off (A/B switch).
inline bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("ENVPOOL_B200_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

// SMs of the current device (132 on an H100 SXM), read once per process: the GPUs of one node
// are the same model.  Sizes grids and CTA caps; never changes what a kernel computes.
inline int device_sm_count() {
  static const int sms = [] {
    int dev = 0, v = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v > 0 ? v : 132;
  }();
  return sms;
}

// CTA size of the single-step kernel: small batches are latency-bound and want many small
// CTAs spread evenly over the SMs, large batches want fewer, fatter CTAs.
// ENVPOOL_B200_STEP_BLOCK overrides (64 | 128 | 256).
inline int step_block_for(int n) {
  static const int forced = [] {
    const char* e = getenv("ENVPOOL_B200_STEP_BLOCK");
    return e ? atoi(e) : 0;
  }();
  if (forced == 64 || forced == 128 || forced == 256) return forced;
  return n <= device_sm_count() * 8 * 128 ? 64 : 128;
}

template <class Env, int kB>
cudaError_t launch_step_b(const LaunchArgs& a) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((a.n + kB - 1) / kB);
  cfg.blockDim = dim3(kB);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = a.stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  // PDL pays off for direct launches (hides part of the launch latency of every step); inside
  // a captured graph the programmatic edges measured slower than plain kernel->kernel edges, so
  // captures keep full serialisation (ENVPOOL_B200_PDL_GRAPH=1 for an A/B run).
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(a.stream, &cap);
  static const bool pdl_in_graph = [] {
    const char* e = getenv("ENVPOOL_B200_PDL_GRAPH");
    return e && e[0] == '1';
  }();
  cfg.numAttrs =
      (pdl_enabled() && (cap == cudaStreamCaptureStatusNone || pdl_in_graph)) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, step_kernel<Env, kB>, a.sv, a.ov,
                            static_cast<const typename Env::Act*>(a.action), a.env_ids, a.n,
                            a.force_reset, a.peers,
                            static_cast<const typename Env::Act*>(a.next_action));
}

template <class Env>
cudaError_t launch_step(const LaunchArgs& a) {
  switch (step_block_for(a.n)) {
    case 64: return launch_step_b<Env, 64>(a);
    case 256: return launch_step_b<Env, 256>(a);
    default: return launch_step_b<Env, 128>(a);
  }
}
template <class Env>
cudaError_t launch_rollout(const LaunchArgs& a) {
  int grid = (a.sv.n_envs + kBlock - 1) / kBlock;
  rollout_kernel<Env><<<grid, kBlock, 0, a.stream>>>(
      a.sv, a.ov, static_cast<const typename Env::Act*>(a.action), a.T);
  return cudaGetLastError();
}

template <class Env>
cudaError_t launch_refill(const LaunchArgs& a) {
  int grid = (a.sv.n_envs + kBlock - 1) / kBlock;
  refill_kernel<Env><<<grid, kBlock, 0, a.stream>>>(a.sv);
  return cudaGetLastError();
}

// family entry points (classic.cu / toytext.cu / mujoco.cu)
launch_fn classic_step_fn(int kind, int precision);
launch_fn classic_refill_fn(int kind, int precision);
launch_fn classic_rollout_fn(int kind, int precision);
launch_fn toytext_step_fn(int kind, int iopt);
launch_fn toytext_rollout_fn(int kind, int iopt);

}  // namespace epb
