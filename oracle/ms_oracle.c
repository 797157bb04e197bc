/* TEST INFRASTRUCTURE ONLY -- CPU restatement of Jumanji's Minesweeper-v0 (the reference's
 * jumanji/minesweeper_env.h driven by core/async_envpool.h in sync mode).
 *
 * Only tests/ and profiles/ load this (through oracle/ms_lib.py); the product (envpool_b200/)
 * never links, imports or calls it.  It is written the plain way on purpose -- the whole
 * 100-entry std::shuffle and a breadth-first Reveal with a queue -- so that it stays independent
 * of the kernel's register-only shuffle and bitboard flood fill.  Parity: pinned bit for bit
 * against the reference's own AsyncEnvPool<MinesweeperEnv> compiled into oracle/_ref
 * (ref_harness/ms_driver.cc), the fixtures recorded from it (tests/golden/minesweeper/) and, for
 * the shuffle, libstdc++ itself (ref_harness/ms_std_rng.cc).
 *
 * Output columns, in the reference's state-key order: info:env_id, info:players.env_id,
 * elapsed_step, done, reward, discount, step_type, trunc, obs:board [10,10],
 * obs:action_mask [10,10], obs:num_mines, obs:step_count.
 */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define CELLS 100
#define WIDTH 10
#define DEFAULT_MINES 10
#define REPLAY_STEPS 32

/* ------------------------------------------------------------------ RNG ---- */
/* std::mt19937 (core/env.h gen_), seeded with one integer as the C++ standard specifies */
typedef struct {
  uint32_t mt[624];
  int idx;
} mso_rng;

static void rng_seed(mso_rng* r, uint32_t seed) {
  r->mt[0] = seed;
  for (int i = 1; i < 624; ++i)
    r->mt[i] = 1812433253u * (r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) + (uint32_t)i;
  r->idx = 624;
}
static uint32_t rng_next(mso_rng* r) {
  if (r->idx >= 624) {
    for (int k = 0; k < 624; ++k) {
      uint32_t y = (r->mt[k] & 0x80000000u) | (r->mt[(k + 1) % 624] & 0x7fffffffu);
      r->mt[k] = r->mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    r->idx = 0;
  }
  uint32_t y = r->mt[r->idx++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}
/* uniform_int_distribution{0, n - 1} on a 32-bit engine: Lemire's method on 32-bit words */
static uint32_t rng_below(mso_rng* r, uint32_t n) {
  uint64_t m = (uint64_t)rng_next(r) * n;
  if ((uint32_t)m < n) {
    uint32_t t = (0u - n) % n;
    while ((uint32_t)m < t) m = (uint64_t)rng_next(r) * n;
  }
  return (uint32_t)(m >> 32);
}
/* std::shuffle of 100 elements (libstdc++ 13): the engine's range fits 100 * 100, so positions
 * are drawn in pairs; 100 is even, so position 1 first takes one draw of its own. */
static void shuffle100(mso_rng* r, int* a) {
  int i = 1, t, j;
  j = (int)rng_below(r, 2);
  t = a[i]; a[i] = a[j]; a[j] = t;
  for (i = 2; i < CELLS; i += 2) {
    uint32_t b1 = (uint32_t)i + 2u;
    uint32_t x = rng_below(r, ((uint32_t)i + 1u) * b1);
    j = (int)(x / b1);
    t = a[i]; a[i] = a[j]; a[j] = t;
    j = (int)(x % b1);
    t = a[i + 1]; a[i + 1] = a[j]; a[j] = t;
  }
}

/* ----------------------------------------------------------------- pool ---- */
typedef struct {
  mso_rng rng;
  int board[CELLS];
  int mine[CELLS];
  int step_count;
  int done;          /* done_, starts true */
  int current_step;  /* Env::current_step_ */
} mso_env;

typedef struct mso_pool {
  int num_envs, max_episode_steps;
  int use_mines, num_mines, use_replay;
  int mines[CELLS];
  int replay[REPLAY_STEPS * CELLS];
  float replay_reward[REPLAY_STEPS];
  int replay_done[REPLAY_STEPS];
  mso_env* envs;
  /* output columns of the last reset / step call */
  int32_t *env_id, *players, *elapsed, *step_type, *board, *num_mines_col, *step_count_col;
  uint8_t *done, *trunc, *mask;
  float *reward, *discount;
} mso_pool;

mso_pool* mso_create(int num_envs, int seed, const int32_t* env_seed, int max_episode_steps) {
  if (num_envs <= 0) return NULL;
  mso_pool* p = (mso_pool*)calloc(1, sizeof(mso_pool));
  size_t n = (size_t)num_envs;
  p->num_envs = num_envs;
  p->max_episode_steps = max_episode_steps > 0 ? max_episode_steps : INT_MAX;
  p->num_mines = DEFAULT_MINES;
  p->envs = (mso_env*)calloc(n, sizeof(mso_env));
  for (int e = 0; e < num_envs; ++e) {
    rng_seed(&p->envs[e].rng, (uint32_t)(env_seed ? env_seed[e] : seed + e));
    p->envs[e].done = 1;
  }
  p->env_id = (int32_t*)calloc(n, 4);
  p->players = (int32_t*)calloc(n, 4);
  p->elapsed = (int32_t*)calloc(n, 4);
  p->step_type = (int32_t*)calloc(n, 4);
  p->board = (int32_t*)calloc(n * CELLS, 4);
  p->num_mines_col = (int32_t*)calloc(n, 4);
  p->step_count_col = (int32_t*)calloc(n, 4);
  p->done = (uint8_t*)calloc(n, 1);
  p->trunc = (uint8_t*)calloc(n, 1);
  p->mask = (uint8_t*)calloc(n * CELLS, 1);
  p->reward = (float*)calloc(n, 4);
  p->discount = (float*)calloc(n, 4);
  return p;
}

void mso_destroy(mso_pool* p) {
  if (!p) return;
  free(p->envs);
  free(p->env_id); free(p->players); free(p->elapsed); free(p->step_type); free(p->board);
  free(p->num_mines_col); free(p->step_count_col); free(p->done); free(p->trunc); free(p->mask);
  free(p->reward); free(p->discount);
  free(p);
}

/* The configuration after the config strings are parsed: mines100 (nonzero = mine; NULL or no
 * mine = random placement of 10), replay boards (32 x 100), rewards and done flags (32 each);
 * replay is on when boards != NULL.  Returns -1 when a replay cell lies outside [-1, 8]. */
int mso_config(mso_pool* p, const int32_t* mines100, const int32_t* boards3200,
               const float* rewards32, const uint8_t* done32) {
  for (int i = 0; boards3200 && i < REPLAY_STEPS * CELLS; ++i)
    if (boards3200[i] < -1 || boards3200[i] > 8) return -1;
  int n = 0;
  for (int c = 0; c < CELLS; ++c) {
    p->mines[c] = mines100 && mines100[c] != 0;
    n += p->mines[c];
  }
  p->use_mines = n > 0;
  p->num_mines = n > 0 ? n : DEFAULT_MINES;
  p->use_replay = boards3200 != NULL;
  for (int i = 0; i < REPLAY_STEPS * CELLS; ++i) p->replay[i] = boards3200 ? boards3200[i] : -1;
  for (int k = 0; k < REPLAY_STEPS; ++k) {
    p->replay_reward[k] = rewards32 ? rewards32[k] : 0.0f;
    p->replay_done[k] = done32 ? done32[k] != 0 : 0;
  }
  return 0;
}

static int adjacent_mines(const mso_env* e, int row, int col) {
  int count = 0;
  for (int dr = -1; dr <= 1; ++dr)
    for (int dc = -1; dc <= 1; ++dc) {
      int r = row + dr, c = col + dc;
      if ((dr || dc) && r >= 0 && r < WIDTH && c >= 0 && c < WIDTH && e->mine[r * WIDTH + c])
        ++count;
    }
  return count;
}
/* breadth-first from the clicked cell: every visited unexplored cell shows its count, and the
 * search goes on from cells with count 0 that hold no mine */
static void reveal(mso_env* e, int row, int col) {
  int queue[CELLS * 9 + 1], head = 0, tail = 0;
  queue[tail++] = row * WIDTH + col;
  while (head < tail) {
    int cell = queue[head++], r = cell / WIDTH, c = cell % WIDTH;
    if (e->board[cell] != -1) continue;
    e->board[cell] = adjacent_mines(e, r, c);
    if (e->board[cell] != 0 || e->mine[cell]) continue;
    for (int dr = -1; dr <= 1; ++dr)
      for (int dc = -1; dc <= 1; ++dc) {
        int rr = r + dr, cc = c + dc;
        if ((dr || dc) && rr >= 0 && rr < WIDTH && cc >= 0 && cc < WIDTH &&
            e->board[rr * WIDTH + cc] == -1)
          queue[tail++] = rr * WIDTH + cc;
      }
  }
}

static void reset_env(mso_pool* p, mso_env* e) {
  for (int c = 0; c < CELLS; ++c) {
    e->board[c] = -1;
    e->mine[c] = 0;
  }
  if (p->use_mines) {
    memcpy(e->mine, p->mines, sizeof(e->mine));
  } else {
    int loc[CELLS];
    for (int c = 0; c < CELLS; ++c) loc[c] = c;
    shuffle100(&e->rng, loc);
    for (int i = 0; i < DEFAULT_MINES; ++i) e->mine[loc[i]] = 1;
  }
  e->step_count = 0;
}

/* one env-step of env `eid` into output row `row`: the worker loop's auto-reset decision
 * (async_envpool.h), MinesweeperEnv::Reset / Step, and Env::Allocate's common columns (env.h) */
static void step_row(mso_pool* p, int eid, int row, int arow, int acol, int force_reset) {
  mso_env* e = &p->envs[eid];
  float reward = 0.0f;
  if (force_reset || e->done) {
    e->current_step = 0;
    reset_env(p, e);
    e->done = 0;
  } else {
    ++e->current_step;
    if (p->use_replay && e->step_count < REPLAY_STEPS) {
      int k = e->step_count++;
      memcpy(e->board, p->replay + (size_t)k * CELLS, sizeof(e->board));
      e->done = p->replay_done[k];
      reward = p->replay_reward[k];
    } else {
      int r = arow < 0 ? 0 : (arow > WIDTH - 1 ? WIDTH - 1 : arow);
      int c = acol < 0 ? 0 : (acol > WIDTH - 1 ? WIDTH - 1 : acol);
      int valid = e->board[r * WIDTH + c] == -1, hit = e->mine[r * WIDTH + c];
      if (valid) {
        reveal(e, r, c);
        reward = hit ? 0.0f : 1.0f;
      }
      ++e->step_count;
      int explored = 0;
      for (int i = 0; i < CELLS; ++i) explored += e->board[i] >= 0;
      e->done = !valid || hit || explored == CELLS - p->num_mines;
    }
  }
  for (int i = 0; i < CELLS; ++i) {
    p->board[(size_t)row * CELLS + i] = e->board[i];
    p->mask[(size_t)row * CELLS + i] = (uint8_t)(e->board[i] == -1);
  }
  p->num_mines_col[row] = p->num_mines;
  p->step_count_col[row] = e->step_count;
  p->env_id[row] = p->players[row] = eid;
  p->elapsed[row] = e->current_step;
  p->done[row] = (uint8_t)e->done;
  p->reward[row] = reward;
  p->discount[row] = e->done ? 0.0f : 1.0f;
  p->step_type[row] = e->current_step == 0 ? 0 : (e->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(e->done && e->current_step >= p->max_episode_steps);
}

/* forced reset / one sync step of the listed envs (NULL = all, in order); row i <-> ids[i];
 * action row i is (row, column) at action[2 i], action[2 i + 1] */
void mso_reset(mso_pool* p, const int32_t* ids, int n) {
  for (int i = 0; i < n; ++i) step_row(p, ids ? ids[i] : i, i, 0, 0, 1);
}
void mso_step(mso_pool* p, const int32_t* action, const int32_t* ids, int n) {
  for (int i = 0; i < n; ++i)
    step_row(p, ids ? ids[i] : i, i, action[2 * i], action[2 * i + 1], 0);
}

/* column k (0..11, the order in this file's header) of the last call */
const void* mso_column(const mso_pool* p, int k) {
  const void* cols[12] = {p->env_id, p->players, p->elapsed, p->done, p->reward, p->discount,
                          p->step_type, p->trunc, p->board, p->mask, p->num_mines_col,
                          p->step_count_col};
  return k >= 0 && k < 12 ? cols[k] : NULL;
}

/* Test hooks: load an engine state (624 words + read position), draw raw words, run the
 * 100-entry shuffle, and overwrite one env's board (cells -1..8) between steps. */
void mso_set_rng(mso_pool* p, int eid, const uint32_t* mt624, int idx) {
  memcpy(p->envs[eid].rng.mt, mt624, sizeof(p->envs[eid].rng.mt));
  p->envs[eid].rng.idx = idx;
}
uint32_t mso_draw(mso_pool* p, int eid) { return rng_next(&p->envs[eid].rng); }
void mso_shuffle(mso_pool* p, int eid, int32_t* out100) {
  int loc[CELLS];
  for (int c = 0; c < CELLS; ++c) loc[c] = c;
  shuffle100(&p->envs[eid].rng, loc);
  for (int c = 0; c < CELLS; ++c) out100[c] = loc[c];
}
void mso_set_board(mso_pool* p, int eid, const int32_t* board100) {
  for (int c = 0; c < CELLS; ++c) p->envs[eid].board[c] = board100[c];
}
