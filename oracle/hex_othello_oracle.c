/* TEST INFRASTRUCTURE ONLY: a plain C restatement of the PGX Hex and Othello envs
 * (pgx/board_games.h) behind the sync step of envpool_b200's engine -- an env that is done
 * resets on its next step -- and the two-player output rows of Env::Allocate(2).  Written from
 * the rules with an int array per board and whole-board scans, independent of the kernels'
 * bitboards (envpool_b200/csrc/pgx.cu): Hex keeps a group id per stone and merges groups on
 * every placement, Othello walks each line cell by cell.  oracle/hex_othello_lib.py drives it;
 * the interface is pgx_oracle.c's, under the prefix hxo_.
 *
 * Columns (hxo_column), rows of the last call: the 13 state keys in the reference's order;
 * info:players.env_id, reward, discount, obs and info:players.id hold two rows per env row
 * (players 0 and 1), the others one. */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { HEX = 0, OTH = 1 };
enum { kMaxCells = 121, kMaxActions = 122 };

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
  int board[kMaxCells];  /* -1 empty, else the colour */
  int group[kMaxCells];  /* Hex: the id of the stone's connected group */
  int mask[kMaxActions];
  int color;           /* the colour to move */
  int current_player;  /* the player to move */
  int done, step;
  int moves;       /* Hex: in-range actions so far (the reference's step_count_) */
  int swap_order;  /* Hex: player p plays colour p ^ swap_order */
  int passed;      /* Othello: the last in-range action was the pass */
} Game;

typedef struct {
  int game, cells, actions, planes, n;
  Game* g;
  /* output columns */
  int32_t *env_id, *players_env_id, *elapsed, *step_type, *board, *current_player, *players_id;
  uint8_t *done, *trunc, *obs, *mask;
  float *reward, *discount;
} Pool;

static const int kDirs8[8][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}, {1, -1}, {-1, 1}, {1, 1}, {-1, -1}};

/* Othello: does `color` capture from cell (r, c) along (dr, dc)?  Walks over the other colour
 * and needs at least one such stone, then one of its own, all on the board.  Returns the
 * distance to that own stone (0: no capture). */
static int oth_line(const Game* g, int r, int c, int dr, int dc, int color) {
  for (int k = 1;; ++k) {
    const int rr = r + dr * k, cc = c + dc * k;
    if (rr < 0 || rr >= 8 || cc < 0 || cc >= 8) return 0;
    const int v = g->board[rr * 8 + cc];
    if (v == color) return k > 1 ? k : 0;
    if (v != 1 - color) return 0;
  }
}

static void update_mask(const Pool* p, Game* g) {
  if (p->game == HEX) {
    for (int i = 0; i < 121; ++i) g->mask[i] = g->board[i] < 0;
    g->mask[121] = g->moves == 1;
    return;
  }
  int any = 0;
  for (int i = 0; i < 64; ++i) {
    g->mask[i] = 0;
    if (g->board[i] >= 0) continue;
    for (int d = 0; d < 8; ++d)
      if (oth_line(g, i / 8, i % 8, kDirs8[d][0], kDirs8[d][1], g->color)) g->mask[i] = 1;
    any |= g->mask[i];
  }
  g->mask[64] = !any;
}

/* Hex: does the group of `cell` reach both of its colour's edges -- rows 0 and 10 for colour 0,
 * columns 0 and 10 for colour 1 (the edges HexEnv::IsTerminal scans)? */
static int hex_joined(const Game* g, int cell) {
  const int color = g->board[cell], id = g->group[cell];
  int a = 0, z = 0;
  for (int i = 0; i < 11; ++i) {
    const int ca = color == 0 ? i : i * 11, cz = color == 0 ? 110 + i : i * 11 + 10;
    a |= g->board[ca] == color && g->group[ca] == id;
    z |= g->board[cz] == color && g->group[cz] == id;
  }
  return a && z;
}

/* Hex: a stone of the colour to move on `cell` (over whatever was there), merged with the groups
 * of the same colour around it; the six neighbours of (r, c) are (r, c -+ 1), (r -+ 1, c),
 * (r + 1, c - 1) and (r - 1, c + 1). */
static void hex_place(Game* g, int cell) {
  static const int nb[6][2] = {{0, -1}, {0, 1}, {-1, 0}, {1, 0}, {1, -1}, {-1, 1}};
  const int r = cell / 11, c = cell % 11, color = g->color;
  g->board[cell] = color;
  g->group[cell] = cell + 1;
  for (int k = 0; k < 6; ++k) {
    const int rr = r + nb[k][0], cc = c + nb[k][1];
    if (rr < 0 || rr >= 11 || cc < 0 || cc >= 11 || g->board[rr * 11 + cc] != color) continue;
    const int old = g->group[rr * 11 + cc];
    for (int i = 0; i < 121; ++i)
      if (g->board[i] == color && g->group[i] == old) g->group[i] = cell + 1;
  }
}

/* Hex: the swap -- the first stone in row-major order, of either colour, leaves its cell and
 * the transposed cell takes a stone of the colour to move; nothing happens on an empty board */
static void hex_swap(Game* g) {
  for (int i = 0; i < 121; ++i) {
    if (g->board[i] < 0) continue;
    const int t = (i % 11) * 11 + i / 11;
    g->board[i] = -1;
    g->board[t] = g->color;
    g->group[t] = t + 1;
    return;
  }
}

static void all_true(const Pool* p, Game* g) {
  for (int a = 0; a < p->actions; ++a) g->mask[a] = 1;
}

static void hex_step(const Pool* p, Game* g, int act, float rw[2]) {
  const int loser = g->current_player;
  const int in_range = act >= 0 && act <= 121;
  const int illegal = !in_range || !g->mask[act];
  const int mover_color = g->color;
  int won = 0;
  if (in_range) {
    if (act < 121) {
      hex_place(g, act);
      won = hex_joined(g, act);
    } else {
      hex_swap(g);
    }
    ++g->moves;
    g->color = g->moves % 2;
    g->current_player = g->color ^ g->swap_order;
  }
  if (illegal) {
    g->done = 1;
    all_true(p, g);
    rw[0] = rw[1] = 1.0f;
    rw[loser] = -1.0f;
    return;
  }
  update_mask(p, g);
  g->done = won;
  if (won) {
    const int winner = mover_color ^ g->swap_order;  /* the player of the colour that moved */
    rw[winner] = 1.0f;
    rw[1 - winner] = -1.0f;
    all_true(p, g);
  }
}

static void oth_step(const Pool* p, Game* g, int act, float rw[2]) {
  const int loser = g->current_player;
  const int in_range = act >= 0 && act <= 64;
  const int illegal = !in_range || !g->mask[act];
  if (in_range) {
    const int me = g->color;
    int both = 0;  /* the action cell holds an opponent stone: it counts for both sides */
    if (act < 64) {
      const int r = act / 8, c = act % 8;
      for (int d = 0; d < 8; ++d) {
        const int k = oth_line(g, r, c, kDirs8[d][0], kDirs8[d][1], me);
        for (int j = 1; j < k; ++j) g->board[(r + kDirs8[d][0] * j) * 8 + c + kDirs8[d][1] * j] = me;
      }
      if (g->board[act] == 1 - me) both = 1;
      else g->board[act] = me;
    }
    int mine = both, theirs = 0, empty = 0;
    for (int i = 0; i < 64; ++i) {
      mine += g->board[i] == me;
      theirs += g->board[i] == 1 - me;
      empty += g->board[i] < 0;
    }
    const int ended = empty == 0 || theirs == 0 || (g->passed && act == 64);
    if (ended && mine != theirs) {
      const int winner = mine > theirs ? g->current_player : 1 - g->current_player;
      rw[winner] = 1.0f;
      rw[1 - winner] = -1.0f;
    }
    g->done = ended;
    g->color = 1 - g->color;
    g->current_player = 1 - g->current_player;
    g->passed = act == 64;
    update_mask(p, g);
  }
  if (illegal) {
    g->done = 1;
    rw[0] = rw[1] = 1.0f;
    rw[loser] = -1.0f;
  }
  if (g->done) all_true(p, g);
}

static void game_reset(const Pool* p, Game* g, float rw[2]) {
  for (int i = 0; i < p->cells; ++i) g->board[i] = -1;
  g->color = 0;
  g->moves = 0;
  g->passed = 0;
  g->done = 0;
  g->step = 0;
  if (p->game == HEX) {
    g->swap_order = (int)(mt_next(&g->rng) & 1u);
    g->current_player = g->swap_order;
  } else {
    g->current_player = (int)(mt_next(&g->rng) & 1u);
    g->board[28] = g->board[35] = 0;  /* colour 0 is the player to move */
    g->board[27] = g->board[36] = 1;
  }
  update_mask(p, g);
  rw[0] = rw[1] = 0.0f;
}

static void write_row(Pool* p, int row, int eid, const float rw[2]) {
  const Game* g = &p->g[eid];
  p->env_id[row] = eid;
  p->elapsed[row] = g->step;
  p->done[row] = (uint8_t)g->done;
  p->step_type[row] = g->step == 0 ? 0 : (g->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(g->done && g->step >= INT_MAX);
  p->current_player[row] = g->current_player;
  /* info:board is relative to the player to move: +1 its stones, -1 the opponent's */
  for (int i = 0; i < p->cells; ++i)
    p->board[row * p->cells + i] = g->board[i] < 0 ? 0 : (g->board[i] == g->color ? 1 : -1);
  for (int a = 0; a < p->actions; ++a) p->mask[row * p->actions + a] = (uint8_t)g->mask[a];
  for (int pl = 0; pl < 2; ++pl) {
    const int r2 = 2 * row + pl;
    p->players_env_id[r2] = eid;
    p->reward[r2] = rw[pl];
    p->discount[r2] = pl == 0 ? (g->done ? 0.0f : 1.0f) : 0.0f;  /* one-element assignment */
    p->players_id[r2] = pl;
    const int my = pl == g->current_player ? g->color : 1 - g->color;
    for (int i = 0; i < p->cells; ++i) {
      uint8_t* o = &p->obs[(r2 * p->cells + i) * p->planes];
      o[0] = g->board[i] == my;
      o[1] = g->board[i] == 1 - my;
      if (p->planes == 4) {  /* Hex: the player's colour is 1; the swap is legal */
        o[2] = my == 1;
        o[3] = g->moves == 1;
      }
    }
  }
}

/* game 0 = Hex, 1 = Othello */
void* hxo_create(int game, int num_envs, int seed, const int32_t* env_seed) {
  if ((game != HEX && game != OTH) || num_envs <= 0) return NULL;
  Pool* p = (Pool*)calloc(1, sizeof(Pool));
  p->game = game;
  p->cells = game == HEX ? 121 : 64;
  p->actions = game == HEX ? 122 : 65;
  p->planes = game == HEX ? 4 : 2;
  p->n = num_envs;
  p->g = (Game*)calloc(num_envs, sizeof(Game));
  for (int e = 0; e < num_envs; ++e) {
    mt_seed(&p->g[e].rng, (uint32_t)(env_seed ? env_seed[e] : seed + e));
    p->g[e].done = 1;
    p->g[e].step = -1;
  }
  const size_t n = (size_t)num_envs;
  p->env_id = (int32_t*)calloc(n, 4);
  p->players_env_id = (int32_t*)calloc(2 * n, 4);
  p->elapsed = (int32_t*)calloc(n, 4);
  p->done = (uint8_t*)calloc(n, 1);
  p->reward = (float*)calloc(2 * n, 4);
  p->discount = (float*)calloc(2 * n, 4);
  p->step_type = (int32_t*)calloc(n, 4);
  p->trunc = (uint8_t*)calloc(n, 1);
  p->obs = (uint8_t*)calloc(2 * n * p->cells * p->planes, 1);
  p->board = (int32_t*)calloc(n * p->cells, 4);
  p->current_player = (int32_t*)calloc(n, 4);
  p->mask = (uint8_t*)calloc(n * p->actions, 1);
  p->players_id = (int32_t*)calloc(2 * n, 4);
  return p;
}

void hxo_destroy(void* h) {
  Pool* p = (Pool*)h;
  if (!p) return;
  void* cols[] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                  p->step_type, p->trunc, p->obs, p->board, p->current_player, p->mask,
                  p->players_id, p->g};
  for (size_t i = 0; i < sizeof(cols) / sizeof(cols[0]); ++i) free(cols[i]);
  free(p);
}

void* hxo_column(void* h, int k) {
  Pool* p = (Pool*)h;
  void* cols[] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                  p->step_type, p->trunc, p->obs, p->board, p->current_player, p->mask,
                  p->players_id};
  return k >= 0 && k < 13 ? cols[k] : NULL;
}

/* forced reset of env_ids[0..n) (NULL: 0..n-1), rows in that order */
void hxo_reset(void* h, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    float rw[2];
    game_reset(p, &p->g[e], rw);
    write_row(p, i, e, rw);
  }
}

/* one sync step of env_ids[0..n) (NULL: 0..n-1) with one action per env row; a done env resets */
void hxo_step(void* h, const int32_t* action, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    Game* g = &p->g[e];
    float rw[2] = {0.0f, 0.0f};
    if (g->done) {
      game_reset(p, g, rw);
    } else {
      ++g->step;
      if (p->game == HEX) hex_step(p, g, action[i], rw);
      else oth_step(p, g, action[i], rw);
    }
    write_row(p, i, e, rw);
  }
}
