/* TEST INFRASTRUCTURE ONLY -- CPU restatement of Jumanji's Game2048-v1 (the reference's
 * jumanji/game2048_env.h driven by core/async_envpool.h in sync mode).
 *
 * Only tests/ and profiles/ load this (through oracle/g2048_lib.py); the product (envpool_b200/)
 * never links, imports or calls it.  Parity: pinned bit for bit against the reference's own
 * AsyncEnvPool<Game2048Env> compiled into oracle/_ref (ref_harness/g2048_driver.cc) and against
 * the fixtures recorded from it (tests/golden/game2048/).  Compile with -ffp-contract=off.
 *
 * Output columns, in the reference's state-key order: info:env_id, info:players.env_id,
 * elapsed_step, done, reward, discount, step_type, trunc, obs:board [4,4], obs:action_mask [4],
 * info:highest_tile.
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ RNG ---- */
/* std::mt19937 (core/env.h gen_), seeded with one integer as the C++ standard specifies */
typedef struct {
  uint32_t mt[624];
  int idx;
} g2o_rng;

static void rng_seed(g2o_rng* r, uint32_t seed) {
  r->mt[0] = seed;
  for (int i = 1; i < 624; ++i)
    r->mt[i] = 1812433253u * (r->mt[i - 1] ^ (r->mt[i - 1] >> 30)) + (uint32_t)i;
  r->idx = 624;
}
static uint32_t rng_next(g2o_rng* r) {
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
/* std::generate_canonical<double, 53>: two words, (w0 + w1 * 2^32) / 2^64, below 1 */
static double rng_canonical(g2o_rng* r) {
  double lo = (double)rng_next(r);
  double hi = (double)rng_next(r);
  double x = (lo + hi * 4294967296.0) / 18446744073709551616.0;
  return x >= 1.0 ? nextafter(1.0, 0.0) : x;
}
/* std::bernoulli_distribution(p): one canonical compared with p */
static int rng_bernoulli(g2o_rng* r, double p) { return rng_canonical(r) < p; }
/* std::uniform_int_distribution<int>(a, b) on a 32-bit engine: Lemire's method */
static int rng_uniform_int(g2o_rng* r, int a, int b) {
  uint32_t range = (uint32_t)b - (uint32_t)a + 1u;
  uint64_t m = (uint64_t)rng_next(r) * range;
  if ((uint32_t)m < range) {
    uint32_t t = (0u - range) % range;
    while ((uint32_t)m < t) m = (uint64_t)rng_next(r) * range;
  }
  return a + (int)(m >> 32);
}

/* ----------------------------------------------------------------- game ---- */
/* Board cell (row, col) is board[row * 4 + col]; directions 0 up, 1 right, 2 down, 3 left.  A
 * line is read so that its position 0 is the edge the tiles slide to. */
static int cell_of(int action, int line, int pos) {
  switch (action) {
    case 0: return pos * 4 + line;
    case 1: return line * 4 + (3 - pos);
    case 2: return (3 - pos) * 4 + line;
    default: return line * 4 + pos;
  }
}
/* MoveLineLeft: drop the gaps, then merge equal neighbours from position 0 on; the line's
 * reward is the float sum of the merged tiles' values in merge order */
static float slide(int* line) {
  int tiles[4], n = 0, out[4] = {0, 0, 0, 0}, m = 0;
  float reward = 0.0f;
  for (int j = 0; j < 4; ++j)
    if (line[j] != 0) tiles[n++] = line[j];
  for (int i = 0; i < n; ++i) {
    if (i + 1 < n && tiles[i] == tiles[i + 1]) {
      out[m] = tiles[i] + 1;
      reward += ldexpf(1.0f, out[m]);
      ++m;
      ++i;
    } else {
      out[m++] = tiles[i];
    }
  }
  memcpy(line, out, sizeof(out));
  return reward;
}
/* Move: every line of the direction, their rewards added for lines 0..3 */
static float move(int* board, int action) {
  float reward = 0.0f;
  for (int i = 0; i < 4; ++i) {
    int line[4];
    for (int j = 0; j < 4; ++j) line[j] = board[cell_of(action, i, j)];
    reward += slide(line);
    for (int j = 0; j < 4; ++j) board[cell_of(action, i, j)] = line[j];
  }
  return reward;
}
static int can_move(const int* board, int action) {
  int moved[16];
  memcpy(moved, board, sizeof(moved));
  move(moved, action);
  return memcmp(moved, board, sizeof(moved)) != 0;
}
static int any_move(const int* board) {
  for (int a = 0; a < 4; ++a)
    if (can_move(board, a)) return 1;
  return 0;
}
/* AddRandomCell's `board_[empty[position_dist(gen_)]] = two_dist(gen_) ? 2 : 1;`: C++17
 * sequences the right operand of `=` first, so the tile value is drawn before its position */
static void random_cell_draw(g2o_rng* r, int n_empty, int* value, int* position) {
  *value = rng_bernoulli(r, 0.1) ? 2 : 1;
  *position = rng_uniform_int(r, 0, n_empty - 1);
}

/* ----------------------------------------------------------------- pool ---- */
typedef struct {
  g2o_rng rng;
  int board[16];
  int done;          /* done_, starts true */
  int current_step;  /* Env::current_step_ (== step_count_ after a step) */
} g2o_env;

typedef struct g2o_pool {
  int num_envs, max_episode_steps, add_random_cell;
  int use_initial, use_replay;
  int initial[16], replay[32 * 16];
  g2o_env* envs;
  /* output columns of the last reset / step call */
  int32_t *env_id, *players, *elapsed, *step_type, *board, *highest;
  uint8_t *done, *trunc, *mask;
  float *reward, *discount;
} g2o_pool;

g2o_pool* g2o_create(int num_envs, int seed, const int32_t* env_seed, int max_episode_steps,
                     int add_random_cell) {
  if (num_envs <= 0) return NULL;
  g2o_pool* p = (g2o_pool*)calloc(1, sizeof(g2o_pool));
  size_t n = (size_t)num_envs;
  p->num_envs = num_envs;
  p->max_episode_steps = max_episode_steps > 0 ? max_episode_steps : INT_MAX;
  p->add_random_cell = add_random_cell != 0;
  p->envs = (g2o_env*)calloc(n, sizeof(g2o_env));
  for (int e = 0; e < num_envs; ++e) {
    rng_seed(&p->envs[e].rng, (uint32_t)(env_seed ? env_seed[e] : seed + e));
    p->envs[e].done = 1;
    p->envs[e].current_step = -1;
  }
  p->env_id = (int32_t*)calloc(n, 4);
  p->players = (int32_t*)calloc(n, 4);
  p->elapsed = (int32_t*)calloc(n, 4);
  p->step_type = (int32_t*)calloc(n, 4);
  p->board = (int32_t*)calloc(n * 16, 4);
  p->highest = (int32_t*)calloc(n, 4);
  p->done = (uint8_t*)calloc(n, 1);
  p->trunc = (uint8_t*)calloc(n, 1);
  p->mask = (uint8_t*)calloc(n * 4, 1);
  p->reward = (float*)calloc(n, 4);
  p->discount = (float*)calloc(n, 4);
  return p;
}

void g2o_destroy(g2o_pool* p) {
  if (!p) return;
  free(p->envs);
  free(p->env_id); free(p->players); free(p->elapsed); free(p->step_type); free(p->board);
  free(p->highest); free(p->done); free(p->trunc); free(p->mask); free(p->reward);
  free(p->discount);
  free(p);
}

/* game2048_initial_board (16 exponents) / game2048_replay_boards (32 x 16), NULL = not
 * configured.  Returns -1 when a cell lies outside [0, 26], else 0. */
int g2o_boards(g2o_pool* p, const int32_t* initial16, const int32_t* replay512) {
  for (int c = 0; initial16 && c < 16; ++c)
    if (initial16[c] < 0 || initial16[c] > 26) return -1;
  for (int c = 0; replay512 && c < 32 * 16; ++c)
    if (replay512[c] < 0 || replay512[c] > 26) return -1;
  p->use_initial = initial16 != NULL;
  p->use_replay = replay512 != NULL;
  for (int c = 0; c < 16; ++c) p->initial[c] = initial16 ? initial16[c] : 0;
  for (int c = 0; c < 32 * 16; ++c) p->replay[c] = replay512 ? replay512[c] : 0;
  return 0;
}

static void add_random_cell(g2o_env* e) {
  int empty[16], n = 0;
  for (int c = 0; c < 16; ++c)
    if (e->board[c] == 0) empty[n++] = c;
  if (n == 0) return;
  int value, position;
  random_cell_draw(&e->rng, n, &value, &position);
  e->board[empty[position]] = value;
}

/* one env-step of env `eid` into output row `row`: the worker loop's auto-reset decision
 * (async_envpool.h), Game2048Env::Reset / Step, and Env::Allocate's common columns (env.h) */
static void step_row(g2o_pool* p, int eid, int row, int action, int force_reset) {
  g2o_env* e = &p->envs[eid];
  float reward = 0.0f;
  if (force_reset || e->done) {
    e->current_step = 0;
    if (p->use_initial) {
      memcpy(e->board, p->initial, sizeof(e->board));
    } else {
      memset(e->board, 0, sizeof(e->board));
      add_random_cell(e); /* whatever add_random_cell says: that flag governs steps only */
    }
  } else {
    ++e->current_step;
    int a = action < 0 ? 0 : (action > 3 ? 3 : action);
    if (can_move(e->board, a)) {
      reward = move(e->board, a);
      if (p->add_random_cell) add_random_cell(e);
    }
    if (p->use_replay && e->current_step <= 32)
      memcpy(e->board, p->replay + (size_t)(e->current_step - 1) * 16, sizeof(e->board));
  }
  e->done = !any_move(e->board);
  int hi = 0;
  for (int c = 0; c < 16; ++c) {
    p->board[(size_t)row * 16 + c] = e->board[c];
    if (e->board[c] > hi) hi = e->board[c];
  }
  for (int a = 0; a < 4; ++a) p->mask[(size_t)row * 4 + a] = (uint8_t)can_move(e->board, a);
  p->highest[row] = hi == 0 ? 1 : (1 << hi);
  p->env_id[row] = p->players[row] = eid;
  p->elapsed[row] = e->current_step;
  p->done[row] = (uint8_t)e->done;
  p->reward[row] = reward;
  p->discount[row] = e->done ? 0.0f : 1.0f;
  p->step_type[row] = e->current_step == 0 ? 0 : (e->done ? 2 : 1);
  p->trunc[row] = (uint8_t)(e->done && e->current_step >= p->max_episode_steps);
}

/* forced reset / one sync step of the listed envs (NULL = all, in order); row i <-> ids[i] */
void g2o_reset(g2o_pool* p, const int32_t* ids, int n) {
  for (int i = 0; i < n; ++i) step_row(p, ids ? ids[i] : i, i, 0, 1);
}
void g2o_step(g2o_pool* p, const int32_t* action, const int32_t* ids, int n) {
  for (int i = 0; i < n; ++i) step_row(p, ids ? ids[i] : i, i, action[i], 0);
}

/* column k (0..10, the order in this file's header) of the last call */
const void* g2o_column(const g2o_pool* p, int k) {
  const void* cols[11] = {p->env_id, p->players, p->elapsed, p->done, p->reward, p->discount,
                          p->step_type, p->trunc, p->board, p->mask, p->highest};
  return k >= 0 && k < 11 ? cols[k] : NULL;
}

/* RNG hooks for the recipe tests: load an engine state (624 words + read position, the
 * representation std::mt19937's operator<< prints), draw raw words, and the distributions */
void g2o_set_rng(g2o_pool* p, int eid, const uint32_t* mt624, int idx) {
  memcpy(p->envs[eid].rng.mt, mt624, sizeof(p->envs[eid].rng.mt));
  p->envs[eid].rng.idx = idx;
}
uint32_t g2o_draw(g2o_pool* p, int eid) { return rng_next(&p->envs[eid].rng); }
int g2o_bernoulli(g2o_pool* p, int eid, double prob) {
  return rng_bernoulli(&p->envs[eid].rng, prob);
}
void g2o_random_cell(g2o_pool* p, int eid, int n_empty, int* value, int* position) {
  random_cell_draw(&p->envs[eid].rng, n_empty, value, position);
}
