/* TEST INFRASTRUCTURE ONLY: a plain C restatement of PGX Chess and GardnerChess
 * (pgx/chess_games.h) behind the sync step of envpool_b200's engine -- an env that is done resets
 * on its next step -- and the two-player output rows of Env::Allocate(2).  Written from the rules
 * with int boards and whole-board scans, independent of the kernel (envpool_b200/csrc/chess.cu),
 * which works on bitboards: here a move is legal when it passes the piece's geometry, path and
 * pawn rules and no enemy piece anywhere on the board attacks the mover's king afterwards; the
 * history is flipped as a whole every step; the position keys are shifted through the whole
 * kMax + 1 entry array and counted there.  The label tables are built by enumerating each plane's
 * direction and distance.  oracle/chess_lib.py drives it; the interface is go_oracle.c's, under
 * the prefix cho_.
 *
 * A label whose target lies off the board moves nothing onto the board: the piece leaves its
 * square, the target reads as empty (DESIGN.md §3).
 *
 * Columns (cho_column), rows of the last call: the state keys in the reference's order (18 for
 * Chess, 16 for GardnerChess); info:players.env_id, reward, discount, obs and info:players.id hold
 * two rows per env row (players 0 and 1), the others one.  With obs off (cho_create's with_obs =
 * 0) the obs column is not filled. */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { kMaxSq = 64, kMaxPlanes = 73, kMaxA = kMaxSq * kMaxPlanes, kHist = 8, kMaxKeys = 513 };
enum { EMPTY = 0, PAWN = 1, KNIGHT = 2, BISHOP = 3, ROOK = 4, QUEEN = 5, KING = 6 };

typedef struct {
  uint32_t mt[624];
  int idx;
} Mt;

static void mt_seed(Mt* m, uint32_t s) {
  m->mt[0] = s;
  for (int i = 1; i < 624; ++i) m->mt[i] = 1812433253u * (m->mt[i - 1] ^ (m->mt[i - 1] >> 30)) + (uint32_t)i;
  m->idx = 624;
}

static uint32_t mt_next(Mt* m) {
  if (m->idx >= 624) {
    for (int i = 0; i < 624; ++i) {
      uint32_t y = (m->mt[i] & 0x80000000u) | (m->mt[(i + 1) % 624] & 0x7fffffffu);
      m->mt[i] = m->mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    m->idx = 0;
  }
  uint32_t v = m->mt[m->idx++];
  v ^= v >> 11;
  v ^= (v << 7) & 0x9d2c5680u;
  v ^= (v << 15) & 0xefc60000u;
  v ^= v >> 18;
  return v;
}

typedef struct {
  Mt rng;
  int board[kMaxSq];          /* the side to move's pieces positive */
  int hist[kHist][kMaxSq];    /* history h: the board h steps back, in the mover's frame */
  uint64_t seen[kMaxKeys];    /* seen[0] the newest key; zero beyond the episode */
  uint8_t mask[kMaxA];
  int rights[2][2];           /* [side: 0 mover, 1 other][0 queen side, 1 king side] */
  int first, color, ep, halfmove, fullmove, moves, done, step;
  int ended;                  /* why the last in-range step ended the game (cho_ended) */
} Game;

typedef struct {
  int chess, S, SQ, P, A, C, kmax, n, with_obs, nkeys;
  int to_of[kMaxSq][kMaxPlanes];   /* plane -> target, -1 off the board */
  int plane_of[kMaxSq][kMaxSq];    /* target -> plane of the plain move, -1 none */
  Game* g;
  int32_t *env_id, *players_env_id, *elapsed, *step_type, *board, *current_player, *en_passant,
      *fullmove, *halfmove, *players_id, *turn;
  uint8_t *done, *trunc, *mask, *castling;
  float *reward, *discount, *obs;
} Pool;

static int iabs(int v) { return v < 0 ? -v : v; }
static int ROW(const Pool* p, int pos) { return pos % p->S; }
static int COL(const Pool* p, int pos) { return pos / p->S; }
static int flip_pos(const Pool* p, int pos) {
  return pos < 0 ? pos : COL(p, pos) * p->S + (p->S - 1 - ROW(p, pos));
}
static int at(const Pool* p, const int* b, int pos) { (void)p; return pos >= 0 ? b[pos] : EMPTY; }

static void make_tables(Pool* p) {
  const int S = p->S, R = S - 1;
  int dr[64], dc[64], n = 0;
  /* the plane directions after the 9 underpromotion planes: files, ranks, diagonals,
   * anti-diagonals (each with distances -R..-1 then 1..R), then the 8 knight jumps */
  for (int kind = 0; kind < 4; ++kind)
    for (int d = -R; d <= R; ++d) {
      if (d == 0) continue;
      dr[n] = kind == 0 ? d : kind == 1 ? 0 : kind == 2 ? d : -d;
      dc[n++] = kind == 0 ? 0 : d;
    }
  const int kn[8][2] = {{-1, -2}, {1, -2}, {-2, -1}, {2, -1}, {-1, 2}, {1, 2}, {-2, 1}, {2, 1}};
  for (int i = 0; i < 8; ++i) {
    dr[n] = kn[i][0];
    dc[n++] = kn[i][1];
  }
  for (int f = 0; f < p->SQ; ++f) {
    for (int t = 0; t < p->SQ; ++t) p->plane_of[f][t] = -1;
    for (int pl = 0; pl < p->P; ++pl) {
      int r, c;
      if (pl < 9) { /* forward, forward + 1 column, forward - 1 column; promotion row only */
        r = ROW(p, f) + 1;
        c = COL(p, f) + (pl % 3 == 0 ? 0 : pl % 3 == 1 ? 1 : -1);
        if (ROW(p, f) != S - 2) r = -1;
      } else {
        r = ROW(p, f) + dr[pl - 9];
        c = COL(p, f) + dc[pl - 9];
      }
      const int on = r >= 0 && r < S && c >= 0 && c < S;
      p->to_of[f][pl] = on ? c * S + r : -1;
      if (on && pl >= 9) p->plane_of[f][c * S + r] = pl;
    }
  }
}

/* can a piece of this type (moving "up" the rows) go from f to t, ignoring what stands there */
static int geometry(const Pool* p, int piece, int f, int t) {
  if (f == t) return 0;
  const int dr = ROW(p, t) - ROW(p, f), dc = COL(p, t) - COL(p, f);
  const int ar = iabs(dr), ac = iabs(dc);
  switch (piece) {
    case PAWN: return (dr == 1 && ac <= 1) || (p->chess && ROW(p, f) == 1 && dr == 2 && dc == 0);
    case KNIGHT: return (ar == 1 && ac == 2) || (ar == 2 && ac == 1);
    case BISHOP: return ar == ac;
    case ROOK: return ar == 0 || ac == 0;
    case QUEEN: return ar == ac || ar == 0 || ac == 0;
    case KING: return ar <= 1 && ac <= 1;
  }
  return 0;
}

static int path_clear(const Pool* p, const int* b, int f, int t) {
  const int dr = ROW(p, t) - ROW(p, f), dc = COL(p, t) - COL(p, f);
  const int sr = (dr > 0) - (dr < 0), sc = (dc > 0) - (dc < 0);
  int r = ROW(p, f) + sr, c = COL(p, f) + sc;
  while (r != ROW(p, t) || c != COL(p, t)) {
    if (b[c * p->S + r] != EMPTY) return 0;
    r += sr;
    c += sc;
  }
  return 1;
}

static int pseudo_legal(const Pool* p, const int* b, int f, int t) {
  if (f < 0 || f >= p->SQ || t < 0 || t >= p->SQ) return 0;
  const int piece = b[f];
  if (piece <= 0 || b[t] > 0 || !geometry(p, piece, f, t)) return 0;
  if ((piece == BISHOP || piece == ROOK || piece == QUEEN || piece == PAWN) &&
      !path_clear(p, b, f, t))
    return 0;
  if (piece == PAWN) {
    if (COL(p, t) == COL(p, f)) return b[t] == EMPTY;
    return b[t] < 0;
  }
  return 1;
}

/* is pos attacked by a piece of the side not to move (negative) */
static int attacked(const Pool* p, const int* b, int pos) {
  for (int q = 0; q < p->SQ; ++q) {
    if (b[q] >= 0) continue;
    const int piece = -b[q];
    if (piece == PAWN) {
      if (ROW(p, q) - ROW(p, pos) == 1 && iabs(COL(p, q) - COL(p, pos)) == 1) return 1;
      continue;
    }
    if (!geometry(p, piece, pos, q)) continue;
    if ((piece == BISHOP || piece == ROOK || piece == QUEEN) && !path_clear(p, b, pos, q)) continue;
    return 1;
  }
  return 0;
}

static int in_check(const Pool* p, const int* b) {
  for (int i = 0; i < p->SQ; ++i)
    if (b[i] == KING) return attacked(p, b, i);
  return 0;
}

/* the move on board b (labels' to = -1: nothing lands); the counters only where given */
static void apply(const Pool* p, Game* g, int* b, int f, int t, int under, int count) {
  int piece = b[f];
  if (p->chess) {
    const int ep_take = g->ep >= 0 && piece == PAWN && g->ep == t;
    if (ep_take && t - 1 >= 0) b[t - 1] = EMPTY;
    const int dbl = piece == PAWN && iabs(t - f) == 2;
    if (count) {
      g->ep = dbl ? (t + f) / 2 : -1;
      const int took = at(p, b, t) < 0 || dbl;
      g->halfmove = took || piece == PAWN ? 0 : g->halfmove + 1;
      g->fullmove += g->color == 1;
    }
    if (piece == KING && f == 32 && t == 16) {
      b[0] = EMPTY;
      b[24] = ROOK;
    }
    if (piece == KING && f == 32 && t == 48) {
      b[56] = EMPTY;
      b[40] = ROOK;
    }
    if (count) {
      g->rights[0][0] = g->rights[0][0] && f != 32 && f != 0;
      g->rights[0][1] = g->rights[0][1] && f != 32 && f != 56;
      g->rights[1][0] = g->rights[1][0] && t != 7;
      g->rights[1][1] = g->rights[1][1] && t != 63;
    }
  } else if (count) {
    const int took = at(p, b, t) < 0;
    g->halfmove = took || piece == PAWN ? 0 : g->halfmove + 1;
    g->fullmove += g->color == 1;
  }
  if (piece == PAWN && ROW(p, f) == p->S - 2 && under < 0) piece = QUEEN;
  if (under >= 0) piece = under == 0 ? ROOK : under == 1 ? BISHOP : KNIGHT;
  b[f] = EMPTY;
  if (t >= 0) b[t] = piece;
}

static int safe_after(const Pool* p, Game* g, int f, int t) {
  int b[kMaxSq];
  memcpy(b, g->board, sizeof(b));
  apply(p, g, b, f, t, -1, 0);
  return !in_check(p, b);
}

static void flip_board(const Pool* p, int* b) {
  int o[kMaxSq];
  for (int i = 0; i < p->SQ; ++i) o[flip_pos(p, i)] = -b[i];
  memcpy(b, o, sizeof(int) * (size_t)p->SQ);
}

static void update_mask(const Pool* p, Game* g) {
  memset(g->mask, 0, (size_t)p->A);
  for (int f = 0; f < p->SQ; ++f) {
    if (g->board[f] <= 0) continue;
    for (int t = 0; t < p->SQ; ++t)
      if (pseudo_legal(p, g->board, f, t) && safe_after(p, g, f, t))
        g->mask[f * p->P + p->plane_of[f][t]] = 1;
  }
  if (p->chess) {
    const int e = g->ep;
    if (e >= 0) {
      const int from[2] = {e - 9, e + 7};
      for (int i = 0; i < 2; ++i) {
        const int f = from[i];
        if (f < 0 || f >= p->SQ || g->board[f] != PAWN || g->board[e - 1] != -PAWN) continue;
        if (p->plane_of[f][e] >= 0 && safe_after(p, g, f, e)) g->mask[f * p->P + p->plane_of[f][e]] = 1;
      }
    }
    const int* b = g->board;
    if (g->rights[0][0] && b[0] == ROOK && b[8] == EMPTY && b[16] == EMPTY && b[24] == EMPTY &&
        b[32] == KING && !attacked(p, b, 16) && !attacked(p, b, 24) && !attacked(p, b, 32))
      g->mask[32 * p->P + p->plane_of[32][16]] = 1;
    if (g->rights[0][1] && b[32] == KING && b[40] == EMPTY && b[48] == EMPTY && b[56] == ROOK &&
        !attacked(p, b, 32) && !attacked(p, b, 40) && !attacked(p, b, 48))
      g->mask[32 * p->P + p->plane_of[32][48]] = 1;
  }
  for (int f = 0; f < p->SQ; ++f) {
    if (ROW(p, f) != p->S - 2 || g->board[f] != PAWN) continue;
    for (int pl = 0; pl < 9; ++pl) {
      const int t = p->to_of[f][pl];
      if (t >= 0 && g->mask[f * p->P + p->plane_of[f][t]]) g->mask[f * p->P + pl] = 1;
    }
  }
}

static uint64_t board_key(const Pool* p, const Game* g) {
  uint64_t key;
  if (p->chess) {
    key = (uint64_t)(g->color + 1) * 131u + (uint64_t)(g->ep + 2);
    for (int s = 0; s < 2; ++s)
      for (int k = 0; k < 2; ++k) key = key * 131u + (uint64_t)g->rights[s][k];
  } else {
    key = (uint64_t)g->color + 1u;
  }
  for (int i = 0; i < p->SQ; ++i) key = key * 1315423911ull + (uint64_t)(g->board[i] + 7);
  return key;
}

static int insufficient(const Pool* p, const int* b) {
  int pieces = 0, prq = 0, bishops = 0, dark = 0;
  for (int i = 0; i < p->SQ; ++i) {
    const int v = iabs(b[i]);
    if (!v) continue;
    ++pieces;
    if (v >= ROOK || v == PAWN) ++prq;
    if (v == BISHOP) {
      ++bishops;
      if (p->chess ? (ROW(p, i) % 2 == COL(p, i) % 2) : (i % 2 == 0)) ++dark;
    }
  }
  prq -= 2;
  return pieces <= 2 || (pieces == 3 && prq == 0) ||
         (pieces == bishops + 2 && (dark == bishops || dark == 0));
}

static void game_reset(const Pool* p, Game* g, float rw[2]) {
  const int S = p->S;
  g->first = (int)(mt_next(&g->rng) & 1u);
  g->color = 0;
  /* rook, knight, bishop, queen, king (, bishop, knight, rook) by column */
  const int back8[8] = {ROOK, KNIGHT, BISHOP, QUEEN, KING, BISHOP, KNIGHT, ROOK};
  const int back5[5] = {ROOK, KNIGHT, BISHOP, QUEEN, KING};
  for (int c = 0; c < S; ++c)
    for (int r = 0; r < S; ++r) {
      const int back = p->chess ? back8[c] : back5[c];
      g->board[c * S + r] = r == 0 ? back : r == 1 ? PAWN : r == S - 2 ? -PAWN : r == S - 1 ? -back : 0;
    }
  memset(g->hist, 0, sizeof(g->hist));
  memcpy(g->hist[0], g->board, sizeof(g->board));
  for (int s = 0; s < 2; ++s) g->rights[s][0] = g->rights[s][1] = p->chess;
  g->ep = -1;
  memset(g->seen, 0, sizeof(g->seen));
  g->seen[0] = board_key(p, g);
  g->halfmove = 0;
  g->fullmove = 1;
  g->moves = 0;
  g->done = 0;
  g->step = 0;
  rw[0] = rw[1] = 0.0f;
  update_mask(p, g);
}

static void game_step(const Pool* p, Game* g, int act, float rw[2]) {
  const int loser = g->color ^ g->first;
  const int in_range = act >= 0 && act < p->A;
  const int illegal = !in_range || !g->mask[act];
  rw[0] = rw[1] = 0.0f;
  g->ended = 0;
  if (in_range) {
    const int f = act / p->P, pl = act % p->P;
    apply(p, g, g->board, f, p->to_of[f][pl], pl < 9 ? pl / 3 : -1, 1);
    flip_board(p, g->board);
    g->color = 1 - g->color;
    if (p->chess) {
      g->ep = flip_pos(p, g->ep);
      for (int k = 0; k < 2; ++k) {
        const int t = g->rights[0][k];
        g->rights[0][k] = g->rights[1][k];
        g->rights[1][k] = t;
      }
    }
    for (int h = kHist - 1; h > 0; --h) {
      memcpy(g->hist[h], g->hist[h - 1], sizeof(g->hist[h]));
      flip_board(p, g->hist[h]);
    }
    memcpy(g->hist[0], g->board, sizeof(g->board));
    ++g->moves;
    for (int i = p->kmax; i > 0; --i) g->seen[i] = g->seen[i - 1];
    g->seen[0] = board_key(p, g);
    update_mask(p, g);
    int any = 0;
    for (int i = 0; i < p->A; ++i) any |= g->mask[i];
    int reps = -1;
    for (int i = 0; i <= p->kmax; ++i) reps += g->seen[i] == g->seen[0];
    const int check = in_check(p, g->board);
    g->ended = (!any) | (check << 1) | ((g->halfmove >= 100) << 2) |
               (insufficient(p, g->board) << 3) | ((reps >= 2) << 4) | ((g->moves >= p->kmax) << 5);
    g->done = !any || g->halfmove >= 100 || insufficient(p, g->board) || reps >= 2 ||
              g->moves >= p->kmax;
    if (!any && check) {
      const int now = g->color ^ g->first;
      rw[now] = -1.0f;
      rw[1 - now] = 1.0f;
    }
  }
  if (illegal) {
    g->done = 1;
    rw[loser] = -1.0f;
    rw[1 - loser] = 1.0f;
  }
  if (g->done) memset(g->mask, 1, (size_t)p->A);
}

static void write_row(Pool* p, int row, int eid, const float rw[2]) {
  const Game* g = &p->g[eid];
  const int S = p->S, SQ = p->SQ, C = p->C;
  const int cur = g->color ^ g->first;
  p->env_id[row] = eid;
  p->elapsed[row] = g->step;
  p->done[row] = (uint8_t)g->done;
  p->step_type[row] = g->step == 0 ? 0 : (g->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(g->done && g->step >= INT_MAX);
  for (int r = 0; r < S; ++r)
    for (int c = 0; c < S; ++c) p->board[(size_t)row * SQ + r * S + c] = g->board[c * S + (S - 1 - r)];
  p->current_player[row] = cur;
  p->fullmove[row] = g->fullmove;
  p->halfmove[row] = g->halfmove;
  p->turn[row] = g->color;
  memcpy(&p->mask[(size_t)row * p->A], g->mask, (size_t)p->A);
  if (p->chess) {
    for (int i = 0; i < 4; ++i) p->castling[(size_t)row * 4 + i] = (uint8_t)g->rights[i / 2][i % 2];
    p->en_passant[row] = g->ep;
  }
  for (int pl = 0; pl < 2; ++pl) {
    const int r2 = 2 * row + pl;
    p->players_env_id[r2] = eid;
    p->reward[r2] = rw[pl];
    p->discount[r2] = pl == 0 ? (g->done ? 0.0f : 1.0f) : 0.0f;  /* one-element assignment */
    p->players_id[r2] = pl;
    if (!p->with_obs) continue;
    const int mine = pl == cur;
    int view[kHist][kMaxSq];
    for (int h = 0; h < kHist; ++h) {
      memcpy(view[h], g->hist[h], sizeof(view[h]));
      if (!mine) flip_board(p, view[h]);
    }
    int rights[4];
    for (int i = 0; i < 4; ++i) rights[i] = mine ? g->rights[i / 2][i % 2] : g->rights[1 - i / 2][i % 2];
    for (int r = 0; r < S; ++r)
      for (int c = 0; c < S; ++c) {
        float* o = &p->obs[(((size_t)r2 * S + r) * S + c) * C];
        const int pos = c * S + (S - 1 - r);
        int ch = 0;
        for (int h = 0; h < kHist; ++h) {
          for (int k = 1; k <= 6; ++k) o[ch++] = view[h][pos] == k ? 1.0f : 0.0f;
          for (int k = 1; k <= 6; ++k) o[ch++] = view[h][pos] == -k ? 1.0f : 0.0f;
          o[ch++] = 1.0f;
          o[ch++] = 0.0f;
        }
        o[ch++] = (float)(mine ? g->color : 1 - g->color);
        o[ch++] = (float)g->moves / (float)p->kmax;
        if (p->chess)
          for (int i = 0; i < 4; ++i) o[ch++] = rights[i] ? 1.0f : 0.0f;
        o[ch++] = (float)g->halfmove / 100.0f;
      }
  }
}

/* game 0 = Chess, 1 = GardnerChess */
void* cho_create(int game, int num_envs, int seed, const int32_t* env_seed, int with_obs) {
  if ((game != 0 && game != 1) || num_envs <= 0) return NULL;
  Pool* p = (Pool*)calloc(1, sizeof(Pool));
  p->chess = game == 0;
  p->S = p->chess ? 8 : 5;
  p->SQ = p->S * p->S;
  p->P = p->chess ? 73 : 49;
  p->A = p->SQ * p->P;
  p->C = p->chess ? 119 : 115;
  p->kmax = p->chess ? 512 : 256;
  p->n = num_envs;
  p->with_obs = with_obs;
  p->nkeys = p->chess ? 18 : 16;
  make_tables(p);
  p->g = (Game*)calloc((size_t)num_envs, sizeof(Game));
  for (int e = 0; e < num_envs; ++e) {
    mt_seed(&p->g[e].rng, (uint32_t)(env_seed ? env_seed[e] : seed + e));
    p->g[e].done = 1;
    p->g[e].step = -1;
  }
  const size_t n = (size_t)num_envs, SQ = (size_t)p->SQ;
  p->env_id = (int32_t*)calloc(n, 4);
  p->players_env_id = (int32_t*)calloc(2 * n, 4);
  p->elapsed = (int32_t*)calloc(n, 4);
  p->done = (uint8_t*)calloc(n, 1);
  p->reward = (float*)calloc(2 * n, 4);
  p->discount = (float*)calloc(2 * n, 4);
  p->step_type = (int32_t*)calloc(n, 4);
  p->trunc = (uint8_t*)calloc(n, 1);
  p->obs = (float*)calloc(with_obs ? 2 * n * SQ * (size_t)p->C : 1, 4);
  p->board = (int32_t*)calloc(n * SQ, 4);
  p->castling = (uint8_t*)calloc(4 * n, 1);
  p->current_player = (int32_t*)calloc(n, 4);
  p->en_passant = (int32_t*)calloc(n, 4);
  p->fullmove = (int32_t*)calloc(n, 4);
  p->halfmove = (int32_t*)calloc(n, 4);
  p->mask = (uint8_t*)calloc(n * (size_t)p->A, 1);
  p->players_id = (int32_t*)calloc(2 * n, 4);
  p->turn = (int32_t*)calloc(n, 4);
  return p;
}

static int columns(Pool* p, void** c) {
  if (p->chess) {
    void* cols[18] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                      p->step_type, p->trunc, p->obs, p->board, p->castling, p->current_player,
                      p->en_passant, p->fullmove, p->halfmove, p->mask, p->players_id, p->turn};
    memcpy(c, cols, sizeof(cols));
    return 18;
  }
  void* cols[16] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                    p->step_type, p->trunc, p->obs, p->board, p->current_player, p->fullmove,
                    p->halfmove, p->mask, p->players_id, p->turn};
  memcpy(c, cols, sizeof(cols));
  return 16;
}

void cho_destroy(void* h) {
  Pool* p = (Pool*)h;
  if (!p) return;
  void* c[18];
  columns(p, c);
  free(p->castling);  /* a Chess column only, allocated for both */
  free(p->en_passant);
  for (int k = 0; k < p->nkeys; ++k)
    if (c[k] != p->castling && c[k] != p->en_passant) free(c[k]);
  free(p->g);
  free(p);
}

void* cho_column(void* h, int k) {
  void* c[18];
  const int n = columns((Pool*)h, c);
  return k >= 0 && k < n ? c[k] : NULL;
}

/* forced reset of env_ids[0..n) (NULL: 0..n-1), rows in that order */
void cho_reset(void* h, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    float rw[2];
    game_reset(p, &p->g[e], rw);
    write_row(p, i, e, rw);
  }
}

/* one sync step of env_ids[0..n) (NULL: 0..n-1) with one action per env row; a done env resets */
void cho_step(void* h, const int32_t* action, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    Game* g = &p->g[e];
    float rw[2] = {0.0f, 0.0f};
    if (g->done) {
      game_reset(p, g, rw);
    } else {
      ++g->step;
      game_step(p, g, action[i], rw);
    }
    write_row(p, i, e, rw);
  }
}

/* copy env src's game into env dst (perft: every continuation of a position) */
void cho_copy_env(void* h, int dst, int src) {
  Pool* p = (Pool*)h;
  p->g[dst] = p->g[src];
}

/* the target square of a label, -1 off the board or out of range */
int cho_label_target(void* h, int label) {
  const Pool* p = (const Pool*)h;
  if (label < 0 || label >= p->A) return -1;
  return p->to_of[label / p->P][label % p->P];
}

/* env e's last in-range step: bit 0 no legal move, 1 the player to move is in check, 2 halfmove
 * >= 100, 3 insufficient material, 4 the key's third occurrence, 5 the step limit */
int cho_ended(void* h, int e) { return ((Pool*)h)->g[e].ended; }

/* is square sq of env e's board (the player to move's frame) attacked by the other side */
int cho_attacked(void* h, int e, int sq) {
  const Pool* p = (const Pool*)h;
  return attacked(p, p->g[e].board, sq);
}
