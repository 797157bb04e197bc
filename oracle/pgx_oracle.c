/* TEST INFRASTRUCTURE ONLY: a plain C restatement of the PGX TicTacToe and ConnectFour envs
 * (pgx/board_games.h) behind the sync step of envpool_b200's engine -- an env that is done
 * resets on its next step -- and the two-player output rows of Env::Allocate(2).  Written from
 * the rules with an int array per board and whole-board scans, independent of the kernel's
 * bitboards (envpool_b200/csrc/pgx.cu).  oracle/pgx_lib.py drives it.
 *
 * Columns (pgo_column), rows of the last call: the 13 state keys in the reference's order;
 * info:players.env_id, reward, discount, obs and info:players.id hold two rows per env row
 * (players 0 and 1), the others one. */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { TTT = 0, C4 = 1 };
enum { kMaxCells = 42, kMaxActions = 9 };

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
  int mask[kMaxActions];
  int color, current_player, winner, done, step;
} Game;

typedef struct {
  int game, rows, cols, cells, actions, n;
  Game* g;
  /* output columns */
  int32_t *env_id, *players_env_id, *elapsed, *step_type, *board, *current_player, *players_id;
  uint8_t *done, *trunc, *obs, *mask;
  float *reward, *discount;
} Pool;

static void update_mask(const Pool* p, Game* g) {
  if (p->game == TTT) {
    for (int i = 0; i < 9; ++i) g->mask[i] = g->board[i] < 0;
  } else {
    for (int c = 0; c < 7; ++c) {
      int filled = 0;
      for (int r = 0; r < 6; ++r) filled += g->board[r * 7 + c] >= 0;
      g->mask[c] = filled < 6;
    }
  }
}

static int ttt_won(const Game* g, int color) {
  static const int lines[8][3] = {{0, 1, 2}, {3, 4, 5}, {6, 7, 8}, {0, 3, 6},
                                  {1, 4, 7}, {2, 5, 8}, {0, 4, 8}, {2, 4, 6}};
  for (int l = 0; l < 8; ++l)
    if (g->board[lines[l][0]] == color && g->board[lines[l][1]] == color &&
        g->board[lines[l][2]] == color)
      return 1;
  return 0;
}

/* four in a row anywhere on the board, scanning every cell in four directions */
static int c4_won(const Game* g, int color) {
  static const int dirs[4][2] = {{1, 0}, {0, 1}, {1, 1}, {1, -1}};
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 7; ++c) {
      if (g->board[r * 7 + c] != color) continue;
      for (int d = 0; d < 4; ++d) {
        int k = 1;
        for (; k < 4; ++k) {
          int rr = r + dirs[d][0] * k, cc = c + dirs[d][1] * k;
          if (rr < 0 || rr >= 6 || cc < 0 || cc >= 7 || g->board[rr * 7 + cc] != color) break;
        }
        if (k == 4) return 1;
      }
    }
  return 0;
}

static void game_reset(const Pool* p, Game* g, float rw[2]) {
  for (int i = 0; i < p->cells; ++i) g->board[i] = -1;
  g->color = 0;
  g->current_player = (int)(mt_next(&g->rng) & 1u);
  g->winner = -1;
  g->done = 0;
  g->step = 0;
  update_mask(p, g);
  rw[0] = rw[1] = 0.0f;
}

static void game_step(const Pool* p, Game* g, int act, float rw[2]) {
  const int loser = g->current_player;
  const int in_range = act >= 0 && act < p->actions;
  const int illegal = !in_range || !g->mask[act];
  ++g->step;
  if (in_range) {
    if (p->game == TTT) {
      g->board[act] = g->color;
      g->winner = ttt_won(g, g->color) ? g->color : -1;
    } else {
      int filled = 0;
      for (int r = 0; r < 6; ++r) filled += g->board[r * 7 + act] >= 0;
      if (5 - filled >= 0) g->board[(5 - filled) * 7 + act] = g->color;
      g->winner = c4_won(g, g->color) ? g->color : -1;
    }
    g->color = 1 - g->color;
    g->current_player = 1 - g->current_player;
  }
  rw[0] = rw[1] = 0.0f;
  if (illegal) {
    g->done = 1;
    for (int a = 0; a < p->actions; ++a) g->mask[a] = 1;
    rw[0] = rw[1] = 1.0f;
    rw[loser] = -1.0f;
    return;
  }
  update_mask(p, g);
  int full = 1;
  if (p->game == TTT) {
    for (int i = 0; i < 9; ++i) full &= g->board[i] >= 0;
  } else {
    for (int a = 0; a < 7; ++a) full &= !g->mask[a];
  }
  g->done = g->winner >= 0 || full;
  if (g->done && g->winner >= 0) {
    float cr[2] = {-1.0f, -1.0f};
    cr[g->winner] = 1.0f;
    if (g->current_player == g->color) {
      rw[0] = cr[0];
      rw[1] = cr[1];
    } else {
      rw[0] = cr[1];
      rw[1] = cr[0];
    }
  }
  if (g->done)
    for (int a = 0; a < p->actions; ++a) g->mask[a] = 1;
}

static void write_row(Pool* p, int row, int eid, const float rw[2]) {
  const Game* g = &p->g[eid];
  p->env_id[row] = eid;
  p->elapsed[row] = g->step;
  p->done[row] = (uint8_t)g->done;
  p->step_type[row] = g->step == 0 ? 0 : (g->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(g->done && g->step >= INT_MAX);
  p->current_player[row] = g->current_player;
  for (int i = 0; i < p->cells; ++i) p->board[row * p->cells + i] = g->board[i];
  for (int a = 0; a < p->actions; ++a) p->mask[row * p->actions + a] = (uint8_t)g->mask[a];
  for (int pl = 0; pl < 2; ++pl) {
    const int r2 = 2 * row + pl;
    p->players_env_id[r2] = eid;
    p->reward[r2] = rw[pl];
    p->discount[r2] = pl == 0 ? (g->done ? 0.0f : 1.0f) : 0.0f;  /* one-element assignment */
    p->players_id[r2] = pl;
    const int my = pl == g->current_player ? g->color : 1 - g->color;
    for (int i = 0; i < p->cells; ++i) {
      p->obs[(r2 * p->cells + i) * 2 + 0] = g->board[i] == my;
      p->obs[(r2 * p->cells + i) * 2 + 1] = g->board[i] == 1 - my;
    }
  }
}

void* pgo_create(int game, int num_envs, int seed, const int32_t* env_seed) {
  if ((game != TTT && game != C4) || num_envs <= 0) return NULL;
  Pool* p = (Pool*)calloc(1, sizeof(Pool));
  p->game = game;
  p->rows = game == TTT ? 3 : 6;
  p->cols = game == TTT ? 3 : 7;
  p->cells = p->rows * p->cols;
  p->actions = game == TTT ? 9 : 7;
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
  p->obs = (uint8_t*)calloc(2 * n * p->cells * 2, 1);
  p->board = (int32_t*)calloc(n * p->cells, 4);
  p->current_player = (int32_t*)calloc(n, 4);
  p->mask = (uint8_t*)calloc(n * p->actions, 1);
  p->players_id = (int32_t*)calloc(2 * n, 4);
  return p;
}

void pgo_destroy(void* h) {
  Pool* p = (Pool*)h;
  if (!p) return;
  void* cols[] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                  p->step_type, p->trunc, p->obs, p->board, p->current_player, p->mask,
                  p->players_id, p->g};
  for (size_t i = 0; i < sizeof(cols) / sizeof(cols[0]); ++i) free(cols[i]);
  free(p);
}

void* pgo_column(void* h, int k) {
  Pool* p = (Pool*)h;
  void* cols[] = {p->env_id, p->players_env_id, p->elapsed, p->done, p->reward, p->discount,
                  p->step_type, p->trunc, p->obs, p->board, p->current_player, p->mask,
                  p->players_id};
  return k >= 0 && k < 13 ? cols[k] : NULL;
}

/* forced reset of env_ids[0..n) (NULL: 0..n-1), rows in that order */
void pgo_reset(void* h, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    float rw[2];
    game_reset(p, &p->g[e], rw);
    write_row(p, i, e, rw);
  }
}

/* one sync step of env_ids[0..n) (NULL: 0..n-1) with one action per env row; a done env resets */
void pgo_step(void* h, const int32_t* action, const int32_t* env_ids, int n) {
  Pool* p = (Pool*)h;
  for (int i = 0; i < n; ++i) {
    const int e = env_ids ? env_ids[i] : i;
    Game* g = &p->g[e];
    float rw[2];
    if (g->done) game_reset(p, g, rw);
    else game_step(p, g, action[i], rw);
    write_row(p, i, e, rw);
  }
}

/* the board and turn of env e, for crafted positions: cells -1 / 0 / 1, a legal game state */
void pgo_set_board(void* h, int e, const int32_t* cells, int color, int current_player) {
  Pool* p = (Pool*)h;
  Game* g = &p->g[e];
  for (int i = 0; i < p->cells; ++i) g->board[i] = cells[i];
  g->color = color;
  g->current_player = current_player;
  g->done = 0;
  g->winner = -1;
  if (g->step < 0) g->step = 0;
  update_mask(p, g);
}
