// PGX Go9x9-v1, Go13x13-v1 and Go19x19-v1 (pgx/go.h GoEnv, rules "pgx" / "tromp_taylor"),
// bit-exact with the reference.  Two players per env, like the other PGX kinds (per-player obs,
// reward, discount and info:players.id; common.cuh write_common_pair).
//
// A Go env does not fit in a thread's registers (a 19x19 env keeps 361 chain ids, 8 history
// planes and up to 722 position hashes), so Go has its own kernel, go_kernel below: ONE WARP PER
// ENV.  Every pass of the reference over the board is a loop over cells xy = 32 k + lane, so
// iteration k of such a loop is word k of a bitboard (__ballot_sync), and lane k keeps that word.
// The env's chain-id board is staged in shared memory; pseudo-liberties are per-chain atomics on
// shared memory; the territory fill and the obs planes work on the bitboards.
//
// State (istate, env-major: env e owns words [e NI, (e + 1) NI), W = ceil(S^2 / 32)):
//   [0] step_count_  [1] ko_  [2] consecutive_pass_count_  [3] flags: bit 0 player_order_[0]
//   (player p plays colour p ^ bit 0), bit 1 is_psk_, bit 2 "the last step ended the game"
//   [4..7] the 128-bit hash of the current board (h0 lo, hi, h1 lo, hi)
//   [8, 8 + 16 W) board history: ring slot s = 0..7 holds colour c's stones (c = 0 black, +1; 1
//   white) in words 8 + (2 s + c) W ...; the board after step i sits in slot i % 8, so a step
//   writes one plane and obs plane h reads slot (step_count_ - 1 - h) % 8.  Slots never written in
//   this episode are zero, which is what a history value of 2 shows in obs.
//   [8 + 16 W, + ceil(S^2 / 2)) chain ids, int16 per cell: 0 empty, else +-(id) as board_ holds them
//   [H, H + 8 S^2) hash_history_: 2 S^2 entries of 4 words (h0 lo, hi, h1 lo, hi), H = a multiple
//   of 4.  Only entries [0, step_count_) are read: the reference's zero entries beyond them can
//   only match a board whose 128-bit hash is zero.
// Configuration (config words at the rstate offset, epb_go_config): [0] 1 = configured, [1..2]
// komi as a double (lo, hi), [3] max_terminal_steps resolved (1..2 S^2).  Unconfigured pools play
// with the registered komi 7.5 and 2 S^2 steps.
//
// Pseudo-liberties: the reference sums, per chain, the number, sum and sum of squares of (cell +
// 1) over the (stone, adjacent empty cell) pairs, and calls a chain in atari when sum^2 ==
// n * sum of squares -- true exactly when every entry is the same cell (or there is none), whose
// index is then sum of squares / sum - 1.  The kernel keeps the least and the greatest such cell
// per chain: in atari <=> min >= max, the single liberty = max (-1 when there is none).
#include <climits>
#include <cstring>

#include "common.cuh"
#include "warp.cuh"

namespace epb {

namespace {

constexpr int kGoBlock = 128;  // 4 envs per CTA
constexpr int kGoWarps = kGoBlock / 32;

template <int S>
struct GoGeom {
  static constexpr int A = S * S;                 // cells; actions are 0..A (A = pass)
  static constexpr int W = (A + 31) / 32;         // bitboard words (one per lane k < W)
  static constexpr int kIdWords = (A + 1) / 2;    // int16 chain ids, two per word
  static constexpr int kHist = 8;
  static constexpr int kIds = kHist + 16 * W;
  static constexpr int kHashes = (kIds + kIdWords + 3) / 4 * 4;
  static constexpr int NI = kHashes + 8 * A;      // 2 A hash entries of 4 words
  static constexpr int kObsBytes = 2 * A * 17;    // obs[2][S][S][17] per env row
  static constexpr uint32_t kSwap = 1u, kPsk = 2u, kOver = 4u;
  // Bytes a step moves (bytes_per_env_step): the header, the 16 history words read and one plane
  // written, the chain ids read and written, one hash entry written.  The psk scan's reads
  // (16 bytes per earlier step of the episode) are not counted.
  static constexpr int kStepStateBytes = 2 * 32 + 16 * W * 4 + 2 * W * 4 + 2 * kIdWords * 4 + 16;
};

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// the contribution of a cell holding `sign` (-1, 0, +1) to ComputeHash
__device__ __forceinline__ void cell_key(int sign, int xy, uint64_t& k0, uint64_t& k1) {
  const uint64_t stone = (uint64_t)(sign + 1);
  k0 = splitmix64(stone * 0x100000001b3ull + (uint64_t)xy);
  k1 = splitmix64(stone * 0x9e3779b97f4a7c15ull + (uint64_t)xy * 17ull);
}
__device__ __forceinline__ uint64_t warp_xor(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ int sgn(int v) { return (v > 0) - (v < 0); }

// Bitboards spread over the lanes, word k on lane k: shifts by 0 < k < 32 cells.
__device__ __forceinline__ uint32_t bb_shl(uint32_t w, int k, int lane) {
  uint32_t prev = __shfl_up_sync(kFull, w, 1);
  if (lane == 0) prev = 0u;
  return (w << k) | (prev >> (32 - k));
}
__device__ __forceinline__ uint32_t bb_shr(uint32_t w, int k, int lane) {
  uint32_t next = __shfl_down_sync(kFull, w, 1);
  if (lane == 31) next = 0u;
  return (w >> k) | (next << (32 - k));
}

template <int S>
__device__ __forceinline__ void neighbours(int xy, int (&nb)[4]) {
  const int x = xy / S, y = xy - x * S;  // GoEnv::Adjacent order: up, down, left, right
  nb[0] = x > 0 ? xy - S : -1;
  nb[1] = x + 1 < S ? xy + S : -1;
  nb[2] = y > 0 ? xy - 1 : -1;
  nb[3] = y + 1 < S ? xy + 1 : -1;
}

// One launch = T sync steps of n batch rows (T = 1: the step kernel, env_ids may permute or
// select rows; T > 1: the fused rollout over every env, actions [T, n]).  Warp w of CTA b is
// batch row 4 b + w.
struct GoHiCols {  // env keys 5..9: info:is_psk, consecutive_pass_count, black / white area, players.id
  void* c[kEnvKeys - 5];
};

template <int S>
__global__ void __launch_bounds__(kGoBlock)
go_kernel(StateView sv, OutView ov, GoHiCols hi, const int32_t* __restrict__ action,
          const int32_t* __restrict__ env_ids, int n, int force_reset, int T) {
  using G = GoGeom<S>;
  constexpr int A = G::A, W = G::W;
  __shared__ int16_t s_id_all[kGoWarps][2 * G::kIdWords];
  __shared__ int32_t s_lo_all[kGoWarps][A];   // least liberty per chain; then obs patterns
  __shared__ int32_t s_hi_all[kGoWarps][A];   // greatest liberty per chain
  __shared__ uint32_t s_hist_all[kGoWarps][16 * W];
  __shared__ uint32_t s_mask_all[kGoWarps][W];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kGoWarps + warp;
  if (row >= n) return;  // the whole warp leaves together
  int16_t* s_id = s_id_all[warp];
  int32_t* s_lo = s_lo_all[warp];
  int32_t* s_hi = s_hi_all[warp];
  uint32_t* s_hist = s_hist_all[warp];
  uint32_t* s_mask = s_mask_all[warp];
  const int eid = env_ids ? env_ids[row] : row;

  double komi = 7.5;
  int max_terminal = 2 * A;
  {
    const uint32_t* cw = static_cast<const uint32_t*>(sv.rstate);
    if (cw[0]) {
      komi = __hiloint2double((int)cw[2], (int)cw[1]);
      max_terminal = (int)cw[3];
    }
  }
  // this lane's word of the board / column-0 / column-(S-1) masks
  uint32_t m_board = 0u, m_col0 = 0u, m_colL = 0u;
  for (int b = 0; b < 32; ++b) {
    const int xy = 32 * lane + b;
    if (lane < W && xy < A) {
      const int y = xy % S;
      m_board |= 1u << b;
      m_col0 |= (y == 0 ? 1u : 0u) << b;
      m_colL |= (y == S - 1 ? 1u : 0u) << b;
    }
  }

  uint32_t* st = reinterpret_cast<uint32_t*>(sv.istate) + (int64_t)eid * G::NI;
  uint4* hashes = reinterpret_cast<uint4*>(st + G::kHashes);
  int step = (int)st[0], ko = (int)st[1], passes = (int)st[2];
  uint32_t fl = st[3];
  uint64_t h0 = (uint64_t)st[4] | ((uint64_t)st[5] << 32);
  uint64_t h1 = (uint64_t)st[6] | ((uint64_t)st[7] << 32);
  for (int i = lane; i < 16 * W; i += 32) s_hist[i] = st[G::kHist + i];
  for (int i = lane; i < G::kIdWords; i += 32)
    reinterpret_cast<uint32_t*>(s_id)[i] = st[G::kIds + i];
  int flags = sv.flags[eid];
  __syncwarp();

  // Per-chain least / greatest adjacent empty cell of the board in s_id (CountLiberties).
  auto liberties = [&]() {
    for (int i = lane; i < A; i += 32) {
      s_lo[i] = INT_MAX;
      s_hi[i] = -1;
    }
    __syncwarp();
    for (int xy = lane; xy < A; xy += 32) {
      if (s_id[xy] != 0) continue;
      int nb[4];
      neighbours<S>(xy, nb);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (nb[i] < 0) continue;
        const int v = s_id[nb[i]];
        if (v != 0) {
          const int c = (v < 0 ? -v : v) - 1;
          atomicMin(&s_lo[c], xy);
          atomicMax(&s_hi[c], xy);
        }
      }
    }
    __syncwarp();
  };
  auto in_atari = [&](int v) {
    const int c = (v < 0 ? -v : v) - 1;
    return s_lo[c] >= s_hi[c];
  };
  // UpdateLegalActionMask's test for an empty cell, for the colour with stones of sign `my`
  auto adj_ok = [&](int xy, int my) {
    int nb[4];
    neighbours<S>(xy, nb);
    bool ok = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (nb[i] < 0) continue;
      const int v = s_id[nb[i]];
      if (v == 0) {
        ok = true;
      } else {
        const bool at = in_atari(v);
        ok |= (v * my < 0 && at) || (v * my > 0 && !at);
      }
    }
    return ok;
  };

  for (int t = 0; t < T; ++t) {
    const int64_t orow = (int64_t)t * ov.t_stride_rows + row;
    int done = flags & 1, cur = flags >> 1;
    float r0 = 0.0f, r1 = 0.0f;  // players 0 and 1
    bool scored = false;         // a legal move: ColorRewards once the game is over
    if (force_reset || done) {
      // GoEnv::Reset: one mt19937 word, the players swap on its bit 1
      uint32_t word = 0u;
      if (lane == 0) {
        Mt rng(sv, eid);
        word = rng.next();
        rng.save(sv, eid);
      }
      word = __shfl_sync(kFull, word, 0);
      step = 0;
      ko = -1;
      passes = 0;
      fl = (word & 2u) ? G::kSwap : 0u;
      for (int i = lane; i < G::kIdWords; i += 32) reinterpret_cast<uint32_t*>(s_id)[i] = 0u;
      for (int i = lane; i < 16 * W; i += 32) {
        s_hist[i] = 0u;
        st[G::kHist + i] = 0u;
      }
      uint64_t e0 = 0ull, e1 = 0ull;
      for (int xy = lane; xy < A; xy += 32) {
        uint64_t k0, k1;
        cell_key(0, xy, k0, k1);
        e0 ^= k0;
        e1 ^= k1;
      }
      h0 = 0x243f6a8885a308d3ull ^ warp_xor(e0);
      h1 = 0x13198a2e03707344ull ^ warp_xor(e1);
      cur = 0;
      done = 0;
      __syncwarp();
    } else {
      ++cur;
      const int act = action[(int64_t)t * n + row];
      const int color = step & 1;
      const int my = color ? -1 : 1;
      const int mover = color ^ (int)(fl & G::kSwap);  // CurrentPlayer()
      const bool in_range = act >= 0 && act <= A;
      const int ko_prev = ko;
      bool illegal = !in_range;
      if (in_range) {
        // StepGame, legal or not
        liberties();
        ko = -1;
        uint64_t d0 = 0ull, d1 = 0ull;  // this lane's share of the hash change
        if (act < A) {
          illegal = s_id[act] != 0 || act == ko_prev || !adj_ok(act, my);
          passes = 0;
          int nb[4], adj[4];
          bool killed[4];
          neighbours<S>(act, nb);
          bool ko_may = true;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            adj[i] = nb[i] < 0 ? 0 : s_id[nb[i]];
            killed[i] = nb[i] >= 0 && adj[i] * my < 0 && in_atari(adj[i]) &&
                        s_hi[(adj[i] < 0 ? -adj[i] : adj[i]) - 1] == act;
            if (nb[i] >= 0 && adj[i] * my >= 0) ko_may = false;
          }
          int ko_cell = -1;  // the first captured neighbour
#pragma unroll
          for (int i = 3; i >= 0; --i)
            if (killed[i]) ko_cell = nb[i];
          __syncwarp();
          int captured = 0;
          for (int xy = lane; xy < A; xy += 32) {
            const int v = s_id[xy];
            bool cap = false;
#pragma unroll
            for (int i = 0; i < 4; ++i) cap |= killed[i] && v != 0 && v == adj[i];
            if (cap) {
              uint64_t a0, a1, b0, b1;
              cell_key(sgn(v), xy, a0, a1);
              cell_key(0, xy, b0, b1);
              d0 ^= a0 ^ b0;
              d1 ^= a1 ^ b1;
              s_id[xy] = 0;
              ++captured;
            }
          }
          captured = warp_sum(captured);
          __syncwarp();
          const int new_id = (act + 1) * my;
          if (lane == 0) {
            const int old = s_id[act];
            if (sgn(old) != my) {
              uint64_t a0, a1, b0, b1;
              cell_key(sgn(old), act, a0, a1);
              cell_key(my, act, b0, b1);
              d0 ^= a0 ^ b0;
              d1 ^= a1 ^ b1;
            }
            s_id[act] = (int16_t)new_id;
          }
          __syncwarp();
          // MergeAdjacentChains
          int target[4];
          bool merge[4];
          int smallest = act + 1;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            target[i] = nb[i] < 0 ? 0 : s_id[nb[i]];
            merge[i] = nb[i] >= 0 && target[i] * my > 0;
            const int at = target[i] < 0 ? -target[i] : target[i];
            if (merge[i] && at < smallest) smallest = at;
          }
          smallest *= my;
          __syncwarp();
          for (int xy = lane; xy < A; xy += 32) {
            const int v = s_id[xy];
            bool m = v == new_id;
#pragma unroll
            for (int i = 0; i < 4; ++i) m |= merge[i] && v == target[i];
            if (m) s_id[xy] = (int16_t)smallest;
          }
          ko = ko_may && captured == 1 ? ko_cell : -1;
          __syncwarp();
        } else {
          ++passes;
        }
        // UpdateBoardHistory: the new board into ring slot step % 8
        const int slot = step & 7;
        for (int k = 0; k < W; ++k) {
          const int xy = 32 * k + lane;
          const int v = xy < A ? (int)s_id[xy] : 0;
          const uint32_t bw = __ballot_sync(kFull, v > 0), ww = __ballot_sync(kFull, v < 0);
          if (lane == k) {
            s_hist[2 * slot * W + k] = bw;
            s_hist[(2 * slot + 1) * W + k] = ww;
            st[G::kHist + 2 * slot * W + k] = bw;
            st[G::kHist + (2 * slot + 1) * W + k] = ww;
          }
        }
        h0 ^= warp_xor(d0);
        h1 ^= warp_xor(d1);
        if (lane == 0 && step < max_terminal)
          hashes[step] = make_uint4((uint32_t)h0, (uint32_t)(h0 >> 32), (uint32_t)h1,
                                    (uint32_t)(h1 >> 32));
        // IsPsk: the hash just stored occurs again among the entries before it
        bool psk = false;
        if (passes == 0) {
          const int seen = step < max_terminal ? step : max_terminal;
          for (int i0 = 0; i0 < seen; i0 += 32) {
            bool hit = false;
            if (i0 + lane < seen) {
              const uint4 e = hashes[i0 + lane];
              hit = e.x == (uint32_t)h0 && e.y == (uint32_t)(h0 >> 32) &&
                    e.z == (uint32_t)h1 && e.w == (uint32_t)(h1 >> 32);
            }
            if (__any_sync(kFull, hit)) {
              psk = true;
              break;
            }
          }
        }
        fl = psk ? (fl | G::kPsk) : (fl & ~G::kPsk);
        ++step;
        __syncwarp();
      }
      if (illegal) {
        done = 1;
        r0 = mover ? 1.0f : -1.0f;
        r1 = -r0;
      } else {
        done = passes >= 2 || (fl & G::kPsk) || max_terminal <= step;
        scored = true;
      }
    }
    fl = done ? (fl | G::kOver) : (fl & ~G::kOver);
    const int color = step & 1;
    const uint32_t swap = fl & G::kSwap;

    // UpdateLegalActionMask for the colour to move (all true once the game is over)
    if (!(fl & G::kOver)) {
      liberties();
      const int my = color ? -1 : 1;
      for (int k = 0; k < W; ++k) {
        const int xy = 32 * k + lane;
        const bool legal = xy < A && s_id[xy] == 0 && xy != ko && adj_ok(xy, my);
        const uint32_t m = __ballot_sync(kFull, legal);
        if (lane == k) s_mask[k] = m;
      }
      __syncwarp();  // s_mask before the mask write; the liberty reads before obs reuses s_lo
    }
    // AreaScores: stones plus the empty cells no path of empty cells joins to the other colour
    const int newest = (step + 7) & 7;
    const uint32_t bw = lane < W ? s_hist[2 * newest * W + lane] : 0u;
    const uint32_t ww = lane < W ? s_hist[(2 * newest + 1) * W + lane] : 0u;
    const uint32_t empty = m_board & ~(bw | ww);
    auto spread = [&](uint32_t r) {
      return (bb_shl(r & ~m_colL, 1, lane) | bb_shr(r & ~m_col0, 1, lane) | bb_shl(r, S, lane) |
              bb_shr(r, S, lane)) & m_board;
    };
    uint32_t from_w = spread(ww) & empty, from_b = spread(bw) & empty;
    for (;;) {
      const uint32_t nw = from_w | (spread(from_w) & empty);
      const uint32_t nbk = from_b | (spread(from_b) & empty);
      const bool changed = nw != from_w || nbk != from_b;
      from_w = nw;
      from_b = nbk;
      if (!__any_sync(kFull, changed)) break;
    }
    const int black_area = warp_sum(__popc(bw) + __popc(empty & ~from_w));
    const int white_area = warp_sum(__popc(ww) + __popc(empty & ~from_b));
    if (scored && done) {
      // ColorRewards of a game that ended without an illegal move
      float c0 = (double)black_area - komi > (double)white_area ? 1.0f : -1.0f;
      float c1 = -c0;
      if (fl & G::kPsk) {
        c0 = color == 0 ? 1.0f : -1.0f;
        c1 = -c0;
      }
      r0 = swap ? c1 : c0;  // player p plays colour p ^ swap
      r1 = swap ? c0 : c1;
    }
    flags = (cur << 1) | done;

    // outputs
    if (lane == 0) {
      StepOut so;
      so.reward = r0;
      so.extra = r1;
      write_common_pair(ov, orow, eid + sv.env_id_offset, cur, done, so, sv.max_steps);
      if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[orow] = color ^ (int)swap;
      if (ov.env[4]) static_cast<int32_t*>(ov.env[4])[orow] = ko;
      if (hi.c[0]) static_cast<uint8_t*>(hi.c[0])[orow] = (fl & G::kPsk) ? 1 : 0;
      if (hi.c[1]) static_cast<int32_t*>(hi.c[1])[orow] = passes;
      if (hi.c[2]) static_cast<int32_t*>(hi.c[2])[orow] = black_area;
      if (hi.c[3]) static_cast<int32_t*>(hi.c[3])[orow] = white_area;
      if (hi.c[4]) reinterpret_cast<int2*>(hi.c[4])[orow] = make_int2(0, 1);
    }
    if (ov.env[1]) {
      int32_t* board = static_cast<int32_t*>(ov.env[1]) + orow * A;
      for (int xy = lane; xy < A; xy += 32) board[xy] = sgn(s_id[xy]);
    }
    if (ov.env[3]) {
      const bool over = (fl & G::kOver) != 0;
      warp_write_bytes(static_cast<uint8_t*>(ov.env[3]) + orow * (A + 1), A + 1, lane,
                       [&](int i) -> uint32_t {
                         return over || i == A || ((s_mask[i >> 5] >> (i & 31)) & 1u) ? 1u : 0u;
                       });
    }
    if (ov.env[0]) {
      // player 0's 17 planes of each cell as one word (bit q = plane q): planes 2h / 2h + 1 are
      // history h in the player's / the other colour, plane 16 "the player's colour is 1";
      // player 1's word swaps each pair and flips plane 16
      uint32_t* pat = reinterpret_cast<uint32_t*>(s_lo);
      const uint32_t c0 = swap;  // player 0's colour
      for (int xy = lane; xy < A; xy += 32) {
        uint32_t p = c0 << 16;
#pragma unroll
        for (int h = 0; h < 8; ++h) {
          const int s = (step + 7 - h) & 7;
          const uint32_t mine = (s_hist[(2 * s + c0) * W + (xy >> 5)] >> (xy & 31)) & 1u;
          const uint32_t other = (s_hist[(2 * s + (c0 ^ 1u)) * W + (xy >> 5)] >> (xy & 31)) & 1u;
          p |= (mine << (2 * h)) | (other << (2 * h + 1));
        }
        pat[xy] = p;
      }
      __syncwarp();
      warp_write_bytes(static_cast<uint8_t*>(ov.env[0]) + orow * G::kObsBytes, G::kObsBytes, lane,
                       [&](int i) -> uint32_t {
                         const int pl = i >= A * 17 ? 1 : 0;
                         const int r = i - pl * A * 17, cell = r / 17, q = r - cell * 17;
                         uint32_t p = pat[cell];
                         if (pl) p = (((p & 0x5555u) << 1) | ((p >> 1) & 0x5555u)) | ((p ^ 0x10000u) & 0x10000u);
                         return (p >> q) & 1u;
                       });
    }
    __syncwarp();
  }

  // write back
  for (int i = lane; i < G::kIdWords; i += 32)
    st[G::kIds + i] = reinterpret_cast<const uint32_t*>(s_id)[i];
  if (lane == 0) {
    st[0] = (uint32_t)step;
    st[1] = (uint32_t)ko;
    st[2] = (uint32_t)passes;
    st[3] = fl;
    st[4] = (uint32_t)h0;
    st[5] = (uint32_t)(h0 >> 32);
    st[6] = (uint32_t)h1;
    st[7] = (uint32_t)(h1 >> 32);
    sv.flags[eid] = flags;
  }
}

template <int S>
cudaError_t go_launch_rows(const LaunchArgs& a, const int32_t* env_ids, int n, int force_reset,
                           int T) {
  const int grid = (n + kGoWarps - 1) / kGoWarps;
  GoHiCols hi;
  for (int k = 0; k < kEnvKeys - 5; ++k) hi.c[k] = a.env_hi[k];
  go_kernel<S><<<grid, kGoBlock, 0, a.stream>>>(a.sv, a.ov, hi, static_cast<const int32_t*>(a.action),
                                                  env_ids, n, force_reset, T);
  return cudaGetLastError();
}
template <int S>
cudaError_t go_step(const LaunchArgs& a) {
  return go_launch_rows<S>(a, a.env_ids, a.n, a.force_reset, 1);
}
template <int S>
cudaError_t go_rollout(const LaunchArgs& a) {
  return go_launch_rows<S>(a, nullptr, a.sv.n_envs, 0, a.T);
}
// bytes_per_env_step counts 2 x NI state words for a step; a Go step moves kStepStateBytes of them
template <int S>
KindLaunch go_launch(int, int) {
  using G = GoGeom<S>;
  return KindLaunch{go_step<S>, go_rollout<S>, nullptr, G::kStepStateBytes - 2 * 4 * G::NI, false};
}

template <int S>
KindDesc go_desc(int kind) {
  using G = GoGeom<S>;
  return KindDesc{
      .kind = kind,
      .keys = {{"obs", EPB_BOOL, 3, {S, S, 17}, true}, {"info:board", EPB_I32, 2, {S, S}},
               {"info:current_player", EPB_I32, 0, {}},
               {"info:legal_action_mask", EPB_BOOL, 1, {G::A + 1}}, {"info:ko", EPB_I32, 0, {}},
               {"info:is_psk", EPB_BOOL, 0, {}}, {"info:consecutive_pass_count", EPB_I32, 0, {}},
               {"info:black_area", EPB_I32, 0, {}}, {"info:white_area", EPB_I32, 0, {}},
               {"info:players.id", EPB_I32, 0, {}, true}},
      .action = kDiscreteAction,
      .NI = G::NI,
      .config_words = 4,
      .fp64_only = true,
      .launch = go_launch<S>,
      .players = 2,
  };
}

// pgx/go.h GoEnvFns::StateSpec.  Any iopt is accepted and ignored, and so is the precision.
const KindDesc kGoKinds[] = {go_desc<9>(EPB_GO_9X9), go_desc<13>(EPB_GO_13X13),
                             go_desc<19>(EPB_GO_19X19)};

}  // namespace

const KindDesc* go_kind(int kind) { return find_kind(kGoKinds, kind); }

const char* go_config(int kind, double komi, int32_t max_terminal_steps,
                      std::vector<uint32_t>& words) {
  const int size = kind == EPB_GO_9X9 ? 9 : kind == EPB_GO_13X13 ? 13 : kind == EPB_GO_19X19 ? 19 : 0;
  if (!size) return "not a Go pool";
  if (max_terminal_steps < 0 || max_terminal_steps > 2 * size * size)
    return "Go: max_terminal_steps must lie in [0, 2 * board_size^2]";
  uint64_t bits;
  memcpy(&bits, &komi, sizeof(bits));
  words = {1u, (uint32_t)bits, (uint32_t)(bits >> 32),
           (uint32_t)(max_terminal_steps > 0 ? max_terminal_steps : 2 * size * size)};
  return nullptr;
}

}  // namespace epb
