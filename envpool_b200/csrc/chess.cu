// PGX Chess-v1 and GardnerChess-v1 (pgx/chess_games.h ChessEnv, GardnerChessEnv), bit-exact with
// the reference.  Two players per env, like the other PGX kinds (per-player obs, reward, discount
// and info:players.id; common.cuh write_common_pair).
//
// ONE WARP PER ENV, as go_kernel: chess_kernel<S> serves the 8x8 game (S = 8) and the 5x5 one
// (S = 5); castling and en passant exist only in the 8x8 instantiation.  Squares are numbered as
// the reference numbers them, pos = col * S + row, with the player to move on rows 0, 1 (the
// board is flipped after every move).  Lane l owns the squares l and l + 32.
//   - Legal moves: pseudo-legal destinations by ray walking plus knight, king and pawn steps; a
//     move is legal when, after making it on the bitboards, the mover's king is not attacked
//     (the reference's "pseudo-legal, then not in check").  The mask is a bitset in shared
//     memory, one bit per label from * planes + plane.
//   - The move itself, the flip and the counters run as the reference writes them, whether the
//     label was legal or not.  A label whose target lies off the board (an underpromotion plane
//     from a square not on the promotion row, a ray or knight plane leaving the board) makes the
//     reference read and write board[-1]; here the write is dropped and the read sees an empty
//     square, the rest of the move arithmetic unchanged (DESIGN.md §3).
//   - Position keys are the reference's polynomial keys, computed as one warp sum of per-square
//     terms; the repetition count scans the episode's stored keys.
//   - obs is written as a flat stream of 16-byte (8x8) or 8-byte (5x5) stores per env row, each
//     element computed from (player, square, channel) against the history boards in shared
//     memory.  The history ring stores each board in the frame of the player who was to move
//     then: board h steps back is in the current mover's frame when h is even.
//
// State (istate, env-major: env e owns words [e NI, (e + 1) NI)):
//   [0] step_count_  [1] halfmove_count_  [2] fullmove_count_
//   [3] flags: bit 0 the first player (player p plays colour p ^ bit 0), bit 1 the colour to move,
//       bits 2..5 castling_rights_ [0][0], [0][1], [1][0], [1][1] (8x8)
//   [4] en_passant_ (8x8; -1 none)
//   [8, 8 + 2 BP) history ring: slot s = 0..7 holds BP bytes, the int8 board after step i in
//   slot i % 8 (the reset board is step 0).  Slots older than the episode are never read.
//   [kMask, + MW) the legal-action bitset of the current position (what the next step's action
//   is judged by: one word is read)
//   [kKeys, + 2 (kMax + 1)) position keys, 64-bit: entry i = the key after step i.  Entries
//   [0, step_count_] are the reference's seen_keys_ in reverse order; its zero entries beyond them
//   are counted without being stored (see repetitions below).
#include <climits>
#include <cstring>

#include "common.cuh"
#include "warp.cuh"

namespace epb {

namespace {

constexpr int kChessBlock = 128;  // 4 envs per CTA
constexpr int kChessWarps = kChessBlock / 32;

enum : int { kPawn = 1, kKnight = 2, kBishop = 3, kRook = 4, kQueen = 5, kKing = 6 };

template <int S>
struct ChessGeom {
  static constexpr bool kChess = S == 8;
  static constexpr int SQ = S * S;
  static constexpr int R = S - 1;                       // longest ray
  static constexpr int P = 9 + 8 * R + 8;               // planes: 73 / 49
  static constexpr int A = SQ * P;                      // labels: 4672 / 1225
  static constexpr int C = kChess ? 119 : 115;          // obs channels
  static constexpr int kMax = kChess ? 512 : 256;       // kMaxTerminationSteps
  static constexpr int BP = (SQ + 3) / 4 * 4;           // bytes per stored board
  static constexpr int MW = (A + 31) / 32;              // mask words: 146 / 39
  static constexpr int kBoards = 8;
  static constexpr int kMask = kBoards + 2 * BP;
  static constexpr int kKeys = (kMask + MW + 1) / 2 * 2;  // 8-byte aligned (NI is even)
  static constexpr int NI = kKeys + 2 * (kMax + 1);
  static constexpr int kObs = 2 * SQ * C;               // floats per env row
  static constexpr int kVec = kChess ? 4 : 2;           // floats per obs store (row bytes % 16 / 8)
  // Bytes a step moves (bytes_per_env_step): the header read and written, the 8 history boards
  // read and one written, one mask word read and the bitset written, one key written.  The
  // repetition scan's reads (8 bytes per earlier step of the episode) are not counted.
  static constexpr int kStepStateBytes = 2 * 32 + 9 * BP + 4 + 4 * MW + 8;
};

constexpr uint64_t kKeyMul = 1315423911ull;

__device__ __forceinline__ uint64_t upow(uint64_t b, int e) {
  uint64_t r = 1;
  while (e) {
    if (e & 1) r *= b;
    b *= b;
    e >>= 1;
  }
  return r;
}
__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// Plane of a move by (dr, dc): the rays (dr, 0), (0, d), (d, d), (-d, d) with d = -R..-1, 1..R in
// that order, then the knight jumps.  -1 when (dr, dc) is neither.
template <int S>
__device__ __forceinline__ int plane_of(int dr, int dc) {
  constexpr int R = S - 1;
  const int adr = dr < 0 ? -dr : dr, adc = dc < 0 ? -dc : dc;
  int type, d;
  if (dc == 0 && dr != 0) { type = 0; d = dr; }
  else if (dr == 0 && dc != 0) { type = 1; d = dc; }
  else if (dr == dc && dr != 0) { type = 2; d = dr; }
  else if (dr == -dc && dr != 0) { type = 3; d = dc; }
  else if ((adr == 1 && adc == 2) || (adr == 2 && adc == 1))
    return 9 + 8 * R + (dc > 0 ? 4 : 0) + (adc == 2 ? 0 : 2) + (dr > 0 ? 1 : 0);
  else return -1;
  return 9 + type * 2 * R + (d < 0 ? d + R : d + R - 1);
}
// The target of label (from, plane), -1 off the board, and its underpromotion (-1: none).
template <int S>
__device__ __forceinline__ void label_move(int from, int plane, int& to, int& up) {
  constexpr int R = S - 1;
  const int r0 = from % S, c0 = from / S;
  int dr, dc;
  up = -1;
  if (plane < 9) {
    up = plane / 3;
    const int k = plane % 3;  // forward, forward-right, forward-left
    dr = 1;
    dc = k == 0 ? 0 : k == 1 ? 1 : -1;
    if (r0 != S - 2) { to = -1; return; }
  } else if (plane < 9 + 8 * R) {
    const int type = (plane - 9) / (2 * R), j = (plane - 9) % (2 * R);
    const int d = j < R ? j - R : j - R + 1;
    dr = type == 0 ? d : type == 1 ? 0 : type == 2 ? d : -d;
    dc = type == 0 ? 0 : d;
  } else {
    const int k = plane - 9 - 8 * R;
    dc = (k & 4) ? ((k & 2) ? 1 : 2) : ((k & 2) ? -1 : -2);
    const int adr = (k & 2) ? 2 : 1;
    dr = (k & 1) ? adr : -adr;
  }
  const int r = r0 + dr, c = c0 + dc;
  to = (r >= 0 && r < S && c >= 0 && c < S) ? c * S + r : -1;
}

// Is square sq attacked by the pieces in t* (the side not to move), with occupancy occ?
template <int S>
__device__ __forceinline__ bool attacked(int sq, uint64_t occ, uint64_t tP, uint64_t tN,
                                         uint64_t tBQ, uint64_t tRQ, uint64_t tK) {
  const int r = sq % S, c = sq / S;
  auto at = [&](uint64_t b, int rr, int cc) {
    return rr >= 0 && rr < S && cc >= 0 && cc < S && ((b >> (cc * S + rr)) & 1ull);
  };
  if (at(tP, r + 1, c - 1) || at(tP, r + 1, c + 1)) return true;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int adr = (k & 2) ? 2 : 1, adc = 3 - adr;
    const int dr = (k & 1) ? adr : -adr, dc = (k & 4) ? adc : -adc;
    if (at(tN, r + dr, c + dc)) return true;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int dr = k < 3 ? -1 : k < 5 ? 0 : 1;
    const int dc = k < 3 ? k - 1 : k < 5 ? (k == 3 ? -1 : 1) : k - 6;
    if (at(tK, r + dr, c + dc)) return true;
    const uint64_t slider = (dr != 0 && dc != 0) ? tBQ : tRQ;
    int rr = r + dr, cc = c + dc;
    while (rr >= 0 && rr < S && cc >= 0 && cc < S) {
      const int p = cc * S + rr;
      if ((occ >> p) & 1ull) {
        if ((slider >> p) & 1ull) return true;
        break;
      }
      rr += dr;
      cc += dc;
    }
  }
  return false;
}

// The current position as bitboards (the side to move is "us", its pieces are positive).
struct Bits {
  uint64_t us, them, tP, tN, tBQ, tRQ, tK;
  int ksq;  // the first of our kings (-1: none)
};
template <int S>
__device__ __forceinline__ Bits bits_of(const int8_t* b, int lane) {
  constexpr int SQ = S * S;
  const int v0 = lane < SQ ? b[lane] : 0;
  const int v1 = lane + 32 < SQ ? b[lane + 32] : 0;
  auto bb = [&](bool p0, bool p1) {
    return (uint64_t)__ballot_sync(kFull, p0) | ((uint64_t)__ballot_sync(kFull, p1) << 32);
  };
  Bits x;
  x.us = bb(v0 > 0, v1 > 0);
  x.them = bb(v0 < 0, v1 < 0);
  x.tP = bb(v0 == -kPawn, v1 == -kPawn);
  x.tN = bb(v0 == -kKnight, v1 == -kKnight);
  x.tBQ = bb(v0 == -kBishop || v0 == -kQueen, v1 == -kBishop || v1 == -kQueen);
  x.tRQ = bb(v0 == -kRook || v0 == -kQueen, v1 == -kRook || v1 == -kQueen);
  x.tK = bb(v0 == -kKing, v1 == -kKing);
  const uint64_t k = bb(v0 == kKing, v1 == kKing);
  x.ksq = k ? __ffsll((long long)k) - 1 : -1;
  return x;
}

// The mover's king is safe after moving from -> to (capturing what stands on `to`, and the pawn
// on `cap` for en passant, cap = -1 otherwise).
template <int S>
__device__ __forceinline__ bool safe_after(const Bits& x, int from, int to, int cap, bool king) {
  const uint64_t tb = 1ull << to, keep = ~(tb | (cap >= 0 ? 1ull << cap : 0ull));
  const uint64_t occ = ((x.us | x.them) & ~(1ull << from) & keep) | tb;
  const int k = king ? to : x.ksq;
  if (k < 0) return true;
  return !attacked<S>(k, occ, x.tP & keep, x.tN & keep, x.tBQ & keep, x.tRQ & keep, x.tK & keep);
}

// UpdateLegalActionMask into the bitset s_mask (MW words).  `b` is the board, ep the en-passant
// square, rights bits 2..5 of the flags word.  Returns whether any label is legal.
template <int S>
__device__ bool legal_mask(const int8_t* b, const Bits& x, int ep, uint32_t fl, uint32_t* s_mask,
                           int lane) {
  using G = ChessGeom<S>;
  for (int i = lane; i < G::MW; i += 32) s_mask[i] = 0u;
  __syncwarp();
  auto set = [&](int label) { atomicOr(&s_mask[label >> 5], 1u << (label & 31)); };
#pragma unroll 1
  for (int from = lane; from < G::SQ; from += 32) {
    const int piece = b[from];
    if (piece <= 0) continue;
    const int r0 = from % S, c0 = from / S, base = from * G::P;
    auto try_to = [&](int r, int c, int cap) {
      const int to = c * S + r;
      if (safe_after<S>(x, from, to, cap, piece == kKing)) set(base + plane_of<S>(r - r0, c - c0));
    };
    auto empty = [&](int r, int c) { return b[c * S + r] == 0; };
    auto enemy = [&](int r, int c) { return b[c * S + r] < 0; };
    if (piece == kPawn) {
      if (r0 + 1 < S) {
        if (empty(r0 + 1, c0)) {
          try_to(r0 + 1, c0, -1);
          if (G::kChess && r0 == 1 && empty(r0 + 2, c0)) try_to(r0 + 2, c0, -1);
        }
        if (c0 > 0 && enemy(r0 + 1, c0 - 1)) try_to(r0 + 1, c0 - 1, -1);
        if (c0 + 1 < S && enemy(r0 + 1, c0 + 1)) try_to(r0 + 1, c0 + 1, -1);
      }
    } else if (piece == kKnight || piece == kKing) {
#pragma unroll 1
      for (int k = 0; k < 8; ++k) {
        int dr, dc;
        if (piece == kKnight) {
          const int adr = (k & 2) ? 2 : 1, adc = 3 - adr;
          dr = (k & 1) ? adr : -adr;
          dc = (k & 4) ? adc : -adc;
        } else {
          dr = k < 3 ? -1 : k < 5 ? 0 : 1;
          dc = k < 3 ? k - 1 : k < 5 ? (k == 3 ? -1 : 1) : k - 6;
        }
        const int r = r0 + dr, c = c0 + dc;
        if (r >= 0 && r < S && c >= 0 && c < S && b[c * S + r] <= 0) try_to(r, c, -1);
      }
    } else {
#pragma unroll 1
      for (int k = 0; k < 8; ++k) {
        const int dr = k < 3 ? -1 : k < 5 ? 0 : 1;
        const int dc = k < 3 ? k - 1 : k < 5 ? (k == 3 ? -1 : 1) : k - 6;
        const bool diag = dr != 0 && dc != 0;
        if ((diag && piece == kRook) || (!diag && piece == kBishop)) continue;
        int r = r0 + dr, c = c0 + dc;
        while (r >= 0 && r < S && c >= 0 && c < S) {
          const int v = b[c * S + r];
          if (v > 0) break;
          try_to(r, c, -1);
          if (v < 0) break;
          r += dr;
          c += dc;
        }
      }
    }
  }
  if constexpr (G::kChess) {
    if (lane == 0) {
      // en passant: from ep - 9 and ep + 7, an enemy pawn on ep - 1, the pawn it takes removed
      if (ep >= 0 && ep - 1 >= 0 && b[ep - 1] == -kPawn) {
        const int cand[2] = {ep - 9, ep + 7};
        for (int i = 0; i < 2; ++i) {
          const int from = cand[i];
          if (from < 0 || from >= G::SQ || b[from] != kPawn) continue;
          const int pl = plane_of<S>(ep % S - from % S, ep / S - from / S);
          if (pl >= 0 && safe_after<S>(x, from, ep, ep - 1, false)) set(from * G::P + pl);
        }
      }
      const uint64_t occ = x.us | x.them;
      auto hit = [&](int sq) { return attacked<S>(sq, occ, x.tP, x.tN, x.tBQ, x.tRQ, x.tK); };
      if ((fl & 4u) && b[0] == kRook && b[8] == 0 && b[16] == 0 && b[24] == 0 && b[32] == kKing &&
          !hit(16) && !hit(24) && !hit(32))
        set(32 * G::P + plane_of<S>(0, -2));
      if ((fl & 8u) && b[32] == kKing && b[40] == 0 && b[48] == 0 && b[56] == kRook &&
          !hit(32) && !hit(40) && !hit(48))
        set(32 * G::P + plane_of<S>(0, 2));
    }
  }
  __syncwarp();
  // underpromotions: planes d, d + 3, d + 6 exactly when the pawn's plain move d is legal
  for (int from = lane; from < G::SQ; from += 32) {
    if (from % S != S - 2 || b[from] != kPawn) continue;
    for (int d = 0; d < 3; ++d) {
      const int dc = d == 0 ? 0 : d == 1 ? 1 : -1, c = from / S + dc;
      if (c < 0 || c >= S) continue;
      const int lab = from * G::P + plane_of<S>(1, dc);
      if ((s_mask[lab >> 5] >> (lab & 31)) & 1u) {
        set(from * G::P + d);
        set(from * G::P + d + 3);
        set(from * G::P + d + 6);
      }
    }
  }
  __syncwarp();
  bool any = false;
  for (int i = lane; i < G::MW; i += 32) any |= s_mask[i] != 0u;
  return __any_sync(kFull, any);
}

// env keys 5..9 (8x8: fullmove, halfmove, mask, players.id, turn; 5x5: mask, players.id, turn)
struct ChessHiCols {
  void* c[kEnvKeys - 5];
};

// One launch = T sync steps of n batch rows (T = 1: the step kernel, env_ids may permute or
// select rows; T > 1: the fused rollout over every env, actions [T, n]).  Warp w of CTA b is
// batch row 4 b + w.
template <int S>
__global__ void __launch_bounds__(kChessBlock)
chess_kernel(StateView sv, OutView ov, ChessHiCols hi, const int32_t* __restrict__ action,
             const int32_t* __restrict__ env_ids, int n, int force_reset, int T) {
  using G = ChessGeom<S>;
  constexpr int SQ = G::SQ;
  __shared__ __align__(16) int8_t s_hist_all[kChessWarps][8 * G::BP];
  __shared__ __align__(16) int8_t s_tmp_all[kChessWarps][G::BP];
  __shared__ uint32_t s_mask_all[kChessWarps][G::MW];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * kChessWarps + warp;
  if (row >= n) return;  // the whole warp leaves together
  int8_t* s_hist = s_hist_all[warp];
  int8_t* s_tmp = s_tmp_all[warp];
  uint32_t* s_mask = s_mask_all[warp];
  const int eid = env_ids ? env_ids[row] : row;

  uint32_t* st = reinterpret_cast<uint32_t*>(sv.istate) + (int64_t)eid * G::NI;
  uint64_t* keys = reinterpret_cast<uint64_t*>(st + G::kKeys);
  int step = (int)st[0], half = (int)st[1], full = (int)st[2];
  uint32_t fl = st[3];
  int ep = (int)st[4];
  for (int i = lane; i < 2 * G::BP; i += 32)
    reinterpret_cast<uint32_t*>(s_hist)[i] = st[G::kBoards + i];
  int flags = sv.flags[eid];
  bool mask_in_smem = false;  // s_mask holds the current position's bitset
  bool mask_dirty = false;    // ... and the state does not
  __syncwarp();

  for (int t = 0; t < T; ++t) {
    const int64_t orow = (int64_t)t * ov.t_stride_rows + row;
    int done = flags & 1, cur = flags >> 1;
    float r0 = 0.0f, r1 = 0.0f;  // players 0 and 1
    bool gen = false;            // a position to judge: the mask, then the endings
    if (force_reset || done) {
      // Reset: one mt19937 word, the first player is its bit 0
      uint32_t word = 0u;
      if (lane == 0) {
        Mt rng(sv, eid);
        word = rng.next();
        rng.save(sv, eid);
      }
      word = __shfl_sync(kFull, word, 0);
      step = 0;
      half = 0;
      full = 1;
      ep = -1;
      fl = (word & 1u) | (G::kChess ? 0x3cu : 0u);
      // the initial board: R N B Q K (B N R) by column on row 0, pawns on row 1, the other side
      // mirrored on rows S - 2 and S - 1
      for (int p = lane; p < G::BP; p += 32) {
        const int r = p % S, c = p / S;
        int v = 0;
        if (p < SQ) {
          const int back = c == 0 || c == 7 ? kRook
                           : c == 1 || c == 6 ? kKnight
                           : c == 2 || c == 5 ? kBishop
                           : c == 3 ? kQueen : kKing;
          v = r == 0 ? back : r == 1 ? kPawn : r == S - 2 ? -kPawn : r == S - 1 ? -back : 0;
        }
        s_hist[p] = (int8_t)v;
      }
      __syncwarp();
      for (int i = lane; i < G::BP / 4; i += 32)
        st[G::kBoards + i] = reinterpret_cast<const uint32_t*>(s_hist)[i];
      cur = 0;
      done = 0;
      gen = true;
    } else {
      ++cur;
      const int act = action[(int64_t)t * n + row];
      const int color = (fl >> 1) & 1;
      const int mover = color ^ (int)(fl & 1u);  // current_player_
      const bool in_range = act >= 0 && act < G::A;
      bool legal = false;
      if (in_range) {
        const uint32_t w = mask_in_smem ? s_mask[act >> 5] : st[G::kMask + (act >> 5)];
        legal = (w >> (act & 31)) & 1u;
        // StepGame, legal or not: the move on a copy of the board, then the flip
        const int8_t* src = s_hist + (step & 7) * G::BP;
        int8_t* dst = s_hist + ((step + 1) & 7) * G::BP;
        for (int i = lane; i < G::BP / 4; i += 32)
          reinterpret_cast<uint32_t*>(s_tmp)[i] = reinterpret_cast<const uint32_t*>(src)[i];
        __syncwarp();
        if (lane == 0) {
          const int from = act / G::P;
          int to, up;
          label_move<S>(from, act % G::P, to, up);
          int piece = s_tmp[from];
          const int at_to = to >= 0 ? s_tmp[to] : 0;  // board[-1] reads as empty
          bool captured = at_to < 0;
          if constexpr (G::kChess) {
            if (ep >= 0 && piece == kPawn && ep == to && to - 1 >= 0) s_tmp[to - 1] = 0;
            const int d = to - from;
            const bool dbl = piece == kPawn && (d == 2 || d == -2);
            ep = dbl ? (to + from) / 2 : -1;
            captured = (to >= 0 ? s_tmp[to] : 0) < 0 || dbl;
          }
          half = captured || piece == kPawn ? 0 : half + 1;
          full += color == 1 ? 1 : 0;
          if constexpr (G::kChess) {
            if (piece == kKing && from == 32 && to == 16) {
              s_tmp[0] = 0;
              s_tmp[24] = kRook;
            }
            if (piece == kKing && from == 32 && to == 48) {
              s_tmp[56] = 0;
              s_tmp[40] = kRook;
            }
            uint32_t rr = fl >> 2;
            if (from == 32 || from == 0) rr &= ~1u;
            if (from == 32 || from == 56) rr &= ~2u;
            if (to == 7) rr &= ~4u;
            if (to == 63) rr &= ~8u;
            // the flip swaps the two sides' rights
            fl = (fl & 3u) | (((rr >> 2) & 3u) << 2) | ((rr & 3u) << 4);
            ep = ep < 0 ? ep : (ep / S) * S + (S - 1 - ep % S);
          }
          if (piece == kPawn && from % S == S - 2 && up < 0) piece = kQueen;
          if (up >= 0) piece = up == 0 ? kRook : up == 1 ? kBishop : kKnight;
          s_tmp[from] = 0;
          if (to >= 0) s_tmp[to] = (int8_t)piece;
        }
        half = __shfl_sync(kFull, half, 0);
        full = __shfl_sync(kFull, full, 0);
        fl = __shfl_sync(kFull, fl, 0) ^ 2u;  // the colour to move flips
        ep = __shfl_sync(kFull, ep, 0);
        __syncwarp();
        for (int p = lane; p < G::BP; p += 32)
          dst[p] = p < SQ ? (int8_t)(-s_tmp[(p / S) * S + (S - 1 - p % S)]) : (int8_t)0;
        ++step;
        __syncwarp();
        for (int i = lane; i < G::BP / 4; i += 32)
          st[G::kBoards + (step & 7) * (G::BP / 4) + i] = reinterpret_cast<const uint32_t*>(dst)[i];
      }
      if (!legal) {
        done = 1;
        r0 = mover ? 1.0f : -1.0f;  // IllegalRewards(loser = the player who moved)
        r1 = -r0;
      } else {
        gen = true;
      }
    }

    const int8_t* b = s_hist + (step & 7) * G::BP;
    const int color = (fl >> 1) & 1;
    const int cp = color ^ (int)(fl & 1u);  // current_player_
    if (gen) {
      const Bits x = bits_of<S>(b, lane);
      const bool has_legal = legal_mask<S>(b, x, ep, fl, s_mask, lane);
      mask_in_smem = true;
      mask_dirty = true;
      // the position key (BoardKey) and its repetitions
      uint64_t term = 0;
      for (int p = lane; p < SQ; p += 32)
        term += (uint64_t)(b[p] + 7) * upow(kKeyMul, SQ - 1 - p);
      uint64_t pre;
      if constexpr (G::kChess) {
        pre = (uint64_t)(color + 1) * 131u + (uint64_t)(ep + 2);
#pragma unroll
        for (int i = 0; i < 4; ++i) pre = pre * 131u + (uint64_t)((fl >> (2 + i)) & 1u);
      } else {
        pre = (uint64_t)(color + 1);
      }
      const uint64_t key = pre * upow(kKeyMul, SQ) + warp_sum64(term);
      if (lane == 0) keys[step] = key;
      __syncwarp();
      int seen = 0;
      for (int i0 = 0; i0 <= step; i0 += 32) {
        const bool hit = i0 + lane <= step && keys[i0 + lane] == key;
        seen += __popc(__ballot_sync(kFull, hit));
      }
      if (key == 0ull) seen += G::kMax - step;  // the reference's zero entries beyond step
      // HasInsufficientPieces
      int pieces = 0, prq = 0, bishops = 0, dark = 0;
      for (int p = lane; p < SQ; p += 32) {
        const int v = b[p] < 0 ? -b[p] : b[p];
        if (!v) continue;
        ++pieces;
        prq += v >= kRook || v == kPawn;
        if (v == kBishop) {
          ++bishops;
          dark += G::kChess ? ((p % S) % 2 == (p / S) % 2) : (p % 2 == 0);
        }
      }
      pieces = warp_sum(pieces);
      prq = warp_sum(prq) - 2;
      bishops = warp_sum(bishops);
      dark = warp_sum(dark);
      const bool insufficient = pieces <= 2 || (pieces == 3 && prq == 0) ||
                                (pieces == bishops + 2 && (dark == bishops || dark == 0));
      if (cur > 0) {
        done = !has_legal || half >= 100 || insufficient || seen - 1 >= 2 || step >= G::kMax;
        const bool checked =
            x.ksq >= 0 && attacked<S>(x.ksq, x.us | x.them, x.tP, x.tN, x.tBQ, x.tRQ, x.tK);
        if (!has_legal && checked) {  // checkmate: the player to move loses
          r0 = cp == 0 ? -1.0f : 1.0f;
          r1 = -r0;
        }
      }
    }
    flags = (cur << 1) | done;

    // outputs
    uint32_t rights = (fl >> 2) & 15u;
    if (lane == 0) {
      StepOut so;
      so.reward = r0;
      so.extra = r1;
      write_common_pair(ov, orow, eid + sv.env_id_offset, cur, done, so, sv.max_steps);
      if constexpr (G::kChess) {
        if (ov.env[2]) {
          uint32_t w = 0u;
          for (int i = 0; i < 4; ++i) w |= ((rights >> i) & 1u) << (8 * i);
          static_cast<uint32_t*>(ov.env[2])[orow] = w;
        }
        if (ov.env[3]) static_cast<int32_t*>(ov.env[3])[orow] = cp;
        if (ov.env[4]) static_cast<int32_t*>(ov.env[4])[orow] = ep;
        if (hi.c[0]) static_cast<int32_t*>(hi.c[0])[orow] = full;
        if (hi.c[1]) static_cast<int32_t*>(hi.c[1])[orow] = half;
        if (hi.c[3]) reinterpret_cast<int2*>(hi.c[3])[orow] = make_int2(0, 1);
        if (hi.c[4]) static_cast<int32_t*>(hi.c[4])[orow] = color;
      } else {
        if (ov.env[2]) static_cast<int32_t*>(ov.env[2])[orow] = cp;
        if (ov.env[3]) static_cast<int32_t*>(ov.env[3])[orow] = full;
        if (ov.env[4]) static_cast<int32_t*>(ov.env[4])[orow] = half;
        if (hi.c[1]) reinterpret_cast<int2*>(hi.c[1])[orow] = make_int2(0, 1);
        if (hi.c[2]) static_cast<int32_t*>(hi.c[2])[orow] = color;
      }
    }
    if (ov.env[1]) {  // info:board(row, col) = board[col * S + (S - 1 - row)]
      int32_t* out = static_cast<int32_t*>(ov.env[1]) + orow * SQ;
      for (int i = lane; i < SQ; i += 32) out[i] = b[(i % S) * S + (S - 1 - i / S)];
    }
    void* mask_col = G::kChess ? hi.c[2] : hi.c[0];
    if (mask_col) {
      warp_write_bytes(static_cast<uint8_t*>(mask_col) + orow * G::A, G::A, lane,
                       [&](int i) -> uint32_t {
                         return done || ((s_mask[i >> 5] >> (i & 31)) & 1u) ? 1u : 0u;
                       });
    }
    if (ov.env[0]) {
      // obs[player][row][col][channel]: per history step h, 6 planes of the player's pieces, 6
      // of the other's and the constant repetition planes (1, 0); then the colour, step_count /
      // kMax, (8x8) the four castling rights and halfmove_count / 100.  The other player sees
      // every board flipped, its own colour and the rights swapped.
      const float f_step = (float)step / (float)G::kMax;
      const float f_half = (float)half / 100.0f;
      const uint32_t rights_swapped = ((rights >> 2) & 3u) | ((rights & 3u) << 2);
      auto value = [&](int i) -> float {
        const int pl = i >= SQ * G::C ? 1 : 0;
        const int rem = i - pl * SQ * G::C, cell = rem / G::C, ch = rem - cell * G::C;
        const bool cv = pl == cp;
        if (ch < 112) {
          const int h = ch / 14, q = ch - 14 * h;
          if (q >= 12) return q == 12 ? 1.0f : 0.0f;
          if (h > step) return 0.0f;
          const int r = cell / S, c = cell - r * S;
          const int8_t* hb = s_hist + ((step - h) & 7) * G::BP;
          const bool flip = cv ? (h & 1) : !(h & 1);
          const int v = flip ? -hb[c * S + r] : hb[c * S + (S - 1 - r)];
          return v == (q < 6 ? q + 1 : -(q - 5)) ? 1.0f : 0.0f;
        }
        const int k = ch - 112;
        if (k == 0) return (float)(cv ? color : 1 - color);
        if (k == 1) return f_step;
        if constexpr (G::kChess) {
          if (k < 6) return (float)(((cv ? rights : rights_swapped) >> (k - 2)) & 1u);
        }
        return f_half;
      };
      float* o = static_cast<float*>(ov.env[0]) + orow * G::kObs;
      if constexpr (G::kVec == 4) {
        float4* o4 = reinterpret_cast<float4*>(o);
        for (int v = lane; v < G::kObs / 4; v += 32)
          o4[v] = make_float4(value(4 * v), value(4 * v + 1), value(4 * v + 2), value(4 * v + 3));
      } else {
        float2* o2 = reinterpret_cast<float2*>(o);
        for (int v = lane; v < G::kObs / 2; v += 32) o2[v] = make_float2(value(2 * v), value(2 * v + 1));
      }
    }
    __syncwarp();
  }

  // write back
  if (mask_dirty)
    for (int i = lane; i < G::MW; i += 32) st[G::kMask + i] = s_mask[i];
  if (lane == 0) {
    st[0] = (uint32_t)step;
    st[1] = (uint32_t)half;
    st[2] = (uint32_t)full;
    st[3] = fl;
    st[4] = (uint32_t)ep;
    sv.flags[eid] = flags;
  }
}

template <int S>
cudaError_t chess_launch_rows(const LaunchArgs& a, const int32_t* env_ids, int n, int force_reset,
                              int T) {
  const int grid = (n + kChessWarps - 1) / kChessWarps;
  ChessHiCols hi;
  for (int k = 0; k < kEnvKeys - 5; ++k) hi.c[k] = a.env_hi[k];
  chess_kernel<S><<<grid, kChessBlock, 0, a.stream>>>(
      a.sv, a.ov, hi, static_cast<const int32_t*>(a.action), env_ids, n, force_reset, T);
  return cudaGetLastError();
}
template <int S>
cudaError_t chess_step(const LaunchArgs& a) {
  return chess_launch_rows<S>(a, a.env_ids, a.n, a.force_reset, 1);
}
template <int S>
cudaError_t chess_rollout(const LaunchArgs& a) {
  return chess_launch_rows<S>(a, nullptr, a.sv.n_envs, 0, a.T);
}
// bytes_per_env_step counts 2 x NI state words for a step; a step moves kStepStateBytes of them
template <int S>
KindLaunch chess_launch(int, int) {
  using G = ChessGeom<S>;
  return KindLaunch{chess_step<S>, chess_rollout<S>, nullptr, G::kStepStateBytes - 2 * 4 * G::NI,
                    false};
}

// pgx/chess_games.h ChessEnvFns / GardnerChessEnvFns::StateSpec.  Any iopt is accepted and
// ignored, and so is the precision.
const KindDesc kChessKinds[] = {
    KindDesc{
        .kind = EPB_CHESS,
        .keys = {{"obs", EPB_F32, 3, {8, 8, 119}, true}, {"info:board", EPB_I32, 2, {8, 8}},
                 {"info:castling_rights", EPB_BOOL, 2, {2, 2}},
                 {"info:current_player", EPB_I32, 0, {}}, {"info:en_passant", EPB_I32, 0, {}},
                 {"info:fullmove_count", EPB_I32, 0, {}}, {"info:halfmove_count", EPB_I32, 0, {}},
                 {"info:legal_action_mask", EPB_BOOL, 1, {ChessGeom<8>::A}},
                 {"info:players.id", EPB_I32, 0, {}, true}, {"info:turn", EPB_I32, 0, {}}},
        .action = kDiscreteAction,
        .NI = ChessGeom<8>::NI,
        .fp64_only = true,
        .launch = chess_launch<8>,
        .players = 2,
    },
    KindDesc{
        .kind = EPB_GARDNER_CHESS,
        .keys = {{"obs", EPB_F32, 3, {5, 5, 115}, true}, {"info:board", EPB_I32, 2, {5, 5}},
                 {"info:current_player", EPB_I32, 0, {}}, {"info:fullmove_count", EPB_I32, 0, {}},
                 {"info:halfmove_count", EPB_I32, 0, {}},
                 {"info:legal_action_mask", EPB_BOOL, 1, {ChessGeom<5>::A}},
                 {"info:players.id", EPB_I32, 0, {}, true}, {"info:turn", EPB_I32, 0, {}}},
        .action = kDiscreteAction,
        .NI = ChessGeom<5>::NI,
        .fp64_only = true,
        .launch = chess_launch<5>,
        .players = 2,
    },
};

}  // namespace

const KindDesc* chess_kind(int kind) { return find_kind(kChessKinds, kind); }

}  // namespace epb
