/* TEST INFRASTRUCTURE ONLY: a plain C restatement of PGX Go (pgx/go.h, rules "pgx") behind the
 * sync step of envpool_b200's engine -- an env that is done resets on its next step -- and the
 * two-player output rows of Env::Allocate(2).  Written from the rules with a sign per cell and
 * whole-board flood fills, independent of the kernel (envpool_b200/csrc/go.cu), which keeps the
 * reference's chain ids and per-chain liberty extremes: here a chain is the connected group of a
 * stone, its liberties the set of empty cells next to it, territory the empty regions, the hash
 * recomputed from the whole board, and the superko test scans the whole hash history.
 * oracle/go_lib.py drives it; the interface is pgx_oracle.c's, under the prefix goo_.
 *
 * Columns (goo_column), rows of the last call: the 18 state keys in the reference's order;
 * info:players.env_id, reward, discount, obs and info:players.id hold two rows per env row
 * (players 0 and 1), the others one. */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { kMaxS = 19, kMaxA = kMaxS * kMaxS, kHist = 8, kPlanes = 17, kKeys = 18 };

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
  int8_t board[kMaxA];          /* +1 black (colour 0), -1 white (colour 1), 0 empty */
  int8_t hist[kHist][kMaxA];    /* history h: the board h steps back, 2 before the episode */
  uint64_t (*hashes)[2];        /* 2 S^2 entries, zero beyond the steps played */
  uint8_t mask[kMaxA + 1];
  int moves;                    /* in-range actions (the reference's step_count_) */
  int ko, passes, psk, swap, done, step;
} Game;

typedef struct {
  int S, A, n, max_terminal;
  double komi;
  Game* g;
  int32_t *env_id, *players_env_id, *elapsed, *step_type, *board, *current_player, *ko, *passes,
      *black_area, *white_area, *players_id;
  uint8_t *done, *trunc, *obs, *mask, *psk;
  float *reward, *discount;
} Pool;

static int nbrs(const Pool* p, int xy, int out[4]) {
  const int S = p->S, r = xy / S, c = xy % S;
  int k = 0;
  if (r > 0) out[k++] = xy - S;
  if (r < S - 1) out[k++] = xy + S;
  if (c > 0) out[k++] = xy - 1;
  if (c < S - 1) out[k++] = xy + 1;
  return k;
}

/* the group of the stone on `xy`: in_group[] = 1 on its stones; returns how many distinct empty
 * cells touch it, and one of them in *lib */
static int group_libs(const Pool* p, const int8_t* b, int xy, uint8_t* in_group, int* lib) {
  int stack[kMaxA], top = 0, nlib = 0;
  uint8_t seen_lib[kMaxA];
  memset(in_group, 0, (size_t)p->A);
  memset(seen_lib, 0, (size_t)p->A);
  in_group[xy] = 1;
  stack[top++] = xy;
  *lib = -1;
  while (top) {
    const int c = stack[--top];
    int nb[4];
    const int k = nbrs(p, c, nb);
    for (int i = 0; i < k; ++i) {
      const int q = nb[i];
      if (b[q] == 0) {
        if (!seen_lib[q]) {
          seen_lib[q] = 1;
          ++nlib;
          *lib = q;
        }
      } else if (b[q] == b[xy] && !in_group[q]) {
        in_group[q] = 1;
        stack[top++] = q;
      }
    }
  }
  return nlib;
}

static uint64_t mix(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

static void board_hash(const Pool* p, const int8_t* b, uint64_t h[2]) {
  h[0] = 0x243f6a8885a308d3ull;
  h[1] = 0x13198a2e03707344ull;
  for (int xy = 0; xy < p->A; ++xy) {
    const uint64_t s = (uint64_t)(b[xy] + 1);
    h[0] ^= mix(s * 0x100000001b3ull + (uint64_t)xy);
    h[1] ^= mix(s * 0x9e3779b97f4a7c15ull + (uint64_t)xy * 17ull);
  }
}

/* stones of `sign` plus the empty regions that touch no stone of -sign */
static int area(const Pool* p, const int8_t* b, int sign) {
  uint8_t seen[kMaxA];
  int stack[kMaxA];
  memset(seen, 0, (size_t)p->A);
  int total = 0;
  for (int xy = 0; xy < p->A; ++xy) {
    if (b[xy] == sign) ++total;
    if (b[xy] != 0 || seen[xy]) continue;
    int top = 0, size = 0, enemy = 0;
    seen[xy] = 1;
    stack[top++] = xy;
    while (top) {
      const int c = stack[--top];
      ++size;
      int nb[4];
      const int k = nbrs(p, c, nb);
      for (int i = 0; i < k; ++i) {
        const int q = nb[i];
        if (b[q] == -sign) enemy = 1;
        else if (b[q] == 0 && !seen[q]) {
          seen[q] = 1;
          stack[top++] = q;
        }
      }
    }
    if (!enemy) total += size;
  }
  return total;
}

/* the legal moves of the colour to move: an empty cell other than the ko point with an empty
 * neighbour, or next to a group of its own with two or more liberties, or next to a group of the
 * other colour with at most one; the pass always */
static void update_mask(const Pool* p, Game* g) {
  const int my = (g->moves & 1) ? -1 : 1;
  uint8_t grp[kMaxA];
  for (int xy = 0; xy < p->A; ++xy) {
    int ok = 0;
    if (g->board[xy] == 0 && xy != g->ko) {
      int nb[4];
      const int k = nbrs(p, xy, nb);
      for (int i = 0; i < k && !ok; ++i) {
        const int q = nb[i], v = g->board[q];
        if (v == 0) {
          ok = 1;
        } else {
          int lib;
          const int nl = group_libs(p, g->board, q, grp, &lib);
          ok = v == my ? nl >= 2 : nl <= 1;
        }
      }
    }
    g->mask[xy] = (uint8_t)ok;
  }
  g->mask[p->A] = 1;
}

static void all_true(const Pool* p, Game* g) { memset(g->mask, 1, (size_t)p->A + 1); }

static void game_reset(const Pool* p, Game* g, float rw[2]) {
  memset(g->board, 0, sizeof(g->board));
  memset(g->hist, 2, sizeof(g->hist));
  memset(g->hashes, 0, sizeof(uint64_t) * 2 * 2 * (size_t)p->A);
  g->moves = 0;
  g->ko = -1;
  g->passes = 0;
  g->psk = 0;
  g->done = 0;
  g->step = 0;
  g->swap = (mt_next(&g->rng) & 2u) ? 1 : 0;
  all_true(p, g);
  rw[0] = rw[1] = 0.0f;
}

/* rewards of colours 0 and 1 into players: player q plays colour q ^ swap */
static void to_players(const Game* g, float c0, float c1, float rw[2]) {
  rw[g->swap] = c0;
  rw[g->swap ^ 1] = c1;
}

static void game_step(const Pool* p, Game* g, int act, float rw[2]) {
  const int A = p->A, color = g->moves & 1, my = color ? -1 : 1;
  const int mover = color ^ g->swap;
  const int in_range = act >= 0 && act <= A;
  const int illegal = !in_range || !g->mask[act];
  rw[0] = rw[1] = 0.0f;
  if (in_range) {
    g->ko = -1;
    if (act < A) {
      g->passes = 0;
      int nb[4], dead[4], ndead = 0, first_dead = -1, all_opp = 1;
      const int k = nbrs(p, act, nb);
      uint8_t grp[kMaxA], gone[kMaxA];
      memset(gone, 0, (size_t)A);
      for (int i = 0; i < k; ++i) {
        if (g->board[nb[i]] != -my) all_opp = 0;
        dead[i] = 0;
        if (g->board[nb[i]] == -my) {
          int lib;
          const int nl = group_libs(p, g->board, nb[i], grp, &lib);
          if (nl == 1 && lib == act) {
            dead[i] = 1;
            for (int q = 0; q < A; ++q) gone[q] |= grp[q];
          }
        }
      }
      for (int i = k - 1; i >= 0; --i)  /* nbrs lists up, down, left, right: the first one */
        if (dead[i]) first_dead = nb[i];
      for (int q = 0; q < A; ++q)
        if (gone[q]) {
          g->board[q] = 0;
          ++ndead;
        }
      g->board[act] = (int8_t)my;
      g->ko = all_opp && ndead == 1 ? first_dead : -1;
    } else {
      ++g->passes;
    }
    memmove(g->hist[1], g->hist[0], sizeof(g->hist[0]) * (kHist - 1));
    memcpy(g->hist[0], g->board, sizeof(g->board));
    uint64_t h[2];
    board_hash(p, g->board, h);
    if (g->moves < p->max_terminal) {
      g->hashes[g->moves][0] = h[0];
      g->hashes[g->moves][1] = h[1];
    }
    g->psk = 0;
    if (g->passes == 0) {
      int same = 0;
      for (int i = 0; i < p->max_terminal; ++i)
        same += g->hashes[i][0] == h[0] && g->hashes[i][1] == h[1];
      g->psk = same > 1;
    }
    ++g->moves;
  }
  if (illegal) {
    g->done = 1;
    all_true(p, g);
    rw[mover] = -1.0f;
    rw[mover ^ 1] = 1.0f;
    return;
  }
  update_mask(p, g);
  g->done = g->passes >= 2 || g->psk || g->moves >= p->max_terminal;
  if (g->done) {
    all_true(p, g);
    const int b = area(p, g->board, 1), w = area(p, g->board, -1);
    float c0 = (double)b - p->komi > (double)w ? 1.0f : -1.0f;
    if (g->psk) c0 = (g->moves & 1) == 0 ? 1.0f : -1.0f;  /* the colour that did not repeat */
    to_players(g, c0, -c0, rw);
  }
}

static void write_row(Pool* p, int row, int eid, const float rw[2]) {
  const Game* g = &p->g[eid];
  const int A = p->A, color = g->moves & 1;
  p->env_id[row] = eid;
  p->elapsed[row] = g->step;
  p->done[row] = (uint8_t)g->done;
  p->step_type[row] = g->step == 0 ? 0 : (g->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(g->done && g->step >= INT_MAX);
  p->current_player[row] = color ^ g->swap;
  for (int xy = 0; xy < A; ++xy) p->board[row * A + xy] = g->board[xy];
  memcpy(&p->mask[(size_t)row * (A + 1)], g->mask, (size_t)A + 1);
  p->ko[row] = g->ko;
  p->psk[row] = (uint8_t)g->psk;
  p->passes[row] = g->passes;
  p->black_area[row] = area(p, g->board, 1);
  p->white_area[row] = area(p, g->board, -1);
  for (int pl = 0; pl < 2; ++pl) {
    const int r2 = 2 * row + pl;
    p->players_env_id[r2] = eid;
    p->reward[r2] = rw[pl];
    p->discount[r2] = pl == 0 ? (g->done ? 0.0f : 1.0f) : 0.0f;  /* one-element assignment */
    p->players_id[r2] = pl;
    const int col = pl ^ g->swap, sign = col ? -1 : 1;
    for (int xy = 0; xy < A; ++xy) {
      uint8_t* o = &p->obs[((size_t)r2 * A + xy) * kPlanes];
      for (int h = 0; h < kHist; ++h) {
        o[2 * h] = g->hist[h][xy] == sign;
        o[2 * h + 1] = g->hist[h][xy] == -sign;
      }
      o[16] = col == 1;
    }
  }
}

/* board_size 9, 13 or 19; max_terminal_steps 0 = 2 S^2 */
void* goo_create(int size, int num_envs, int seed, const int32_t* env_seed, double komi,
                 int max_terminal_steps) {
  if ((size != 9 && size != 13 && size != 19) || num_envs <= 0) return NULL;
  Pool* p = (Pool*)calloc(1, sizeof(Pool));
  p->S = size;
  p->A = size * size;
  p->n = num_envs;
  p->komi = komi;
  p->max_terminal = max_terminal_steps > 0 ? max_terminal_steps : 2 * p->A;
  p->g = (Game*)calloc(num_envs, sizeof(Game));
  for (int e = 0; e < num_envs; ++e) {
    mt_seed(&p->g[e].rng, (uint32_t)(env_seed ? env_seed[e] : seed + e));
    p->g[e].hashes = (uint64_t(*)[2])calloc(2 * (size_t)p->A, sizeof(uint64_t[2]));
    p->g[e].done = 1;
    p->g[e].step = -1;
  }
  const size_t n = (size_t)num_envs, A = (size_t)p->A;
  p->env_id = (int32_t*)calloc(n, 4);
  p->players_env_id = (int32_t*)calloc(2 * n, 4);
  p->elapsed = (int32_t*)calloc(n, 4);
  p->done = (uint8_t*)calloc(n, 1);
  p->reward = (float*)calloc(2 * n, 4);
  p->discount = (float*)calloc(2 * n, 4);
  p->step_type = (int32_t*)calloc(n, 4);
  p->trunc = (uint8_t*)calloc(n, 1);
  p->obs = (uint8_t*)calloc(2 * n * A * kPlanes, 1);
  p->board = (int32_t*)calloc(n * A, 4);
  p->current_player = (int32_t*)calloc(n, 4);
  p->mask = (uint8_t*)calloc(n * (A + 1), 1);
  p->ko = (int32_t*)calloc(n, 4);
  p->psk = (uint8_t*)calloc(n, 1);
  p->passes = (int32_t*)calloc(n, 4);
  p->black_area = (int32_t*)calloc(n, 4);
  p->white_area = (int32_t*)calloc(n, 4);
  p->players_id = (int32_t*)calloc(2 * n, 4);
  return p;
}

static void** columns(Pool* p, void** c) {
  void* cols[kKeys] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward,
                       p->discount, p->step_type, p->trunc, p->obs, p->board,
                       p->current_player, p->mask, p->ko, p->psk, p->passes,
                       p->black_area, p->white_area, p->players_id};
  memcpy(c, cols, sizeof(cols));
  return c;
}

void goo_destroy(void* h) {
  Pool* p = (Pool*)h;
  if (!p) return;
  void* c[kKeys];
  columns(p, c);
  for (int k = 0; k < kKeys; ++k) free(c[k]);
  for (int e = 0; e < p->n; ++e) free(p->g[e].hashes);
  free(p->g);
  free(p);
}

void* goo_column(void* h, int k) {
  void* c[kKeys];
  return k >= 0 && k < kKeys ? columns((Pool*)h, c)[k] : NULL;
}

/* forced reset of env_ids[0..n) (NULL: 0..n-1), rows in that order */
void goo_reset(void* h, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    float rw[2];
    game_reset(p, &p->g[e], rw);
    write_row(p, i, e, rw);
  }
}

/* one sync step of env_ids[0..n) (NULL: 0..n-1) with one action per env row; a done env resets */
void goo_step(void* h, const int32_t* action, const int32_t* env_ids, int n) {
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
