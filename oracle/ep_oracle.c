/* TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's batched step() hot
 * path (see ep_oracle.h for who may load this and for the parity status).
 *
 * Every function cites the reference file:line it restates (paths relative to
 * the reference tree's envpool/).  All env arithmetic is double, exactly as the reference;
 * compile with -ffp-contract=off so no FMA contraction changes rounding (the reference
 * is built for baseline x86-64, which has no FMA).
 */
#include "ep_oracle.h"

#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "mjc_oracle.h"

/* ------------------------------------------------------------------ RNG ---- */
/* std::mt19937 as used by Env::gen_ (core/env.h:75,113): MT19937 with the
 * single-integer seeding of the C++ standard (== init_genrand of the 2002 reference
 * code by Matsumoto & Nishimura). */
typedef struct {
  uint32_t mt[624];
  int idx;
  /* std::normal_distribution<double> saved state (bits/random.tcc:1811-1844) */
  int norm_has_saved;
  double norm_saved;
} epo_rng;

static void rng_seed(epo_rng* r, uint32_t seed) {
  r->mt[0] = seed;
  for (int i = 1; i < 624; ++i) {
    uint32_t prev = r->mt[i - 1];
    r->mt[i] = 1812433253u * (prev ^ (prev >> 30)) + (uint32_t)i;
  }
  r->idx = 624;
  r->norm_has_saved = 0;
  r->norm_saved = 0.0;
}

static uint32_t rng_next(epo_rng* r) {
  if (r->idx >= 624) {
    uint32_t* mt = r->mt;
    for (int k = 0; k < 624; ++k) {
      uint32_t y = (mt[k] & 0x80000000u) | (mt[(k + 1) % 624] & 0x7fffffffu);
      mt[k] = mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    r->idx = 0;
  }
  uint32_t y = r->mt[r->idx++];
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

/* std::generate_canonical<double,53>(mt19937): libstdc++ 13 bits/random.tcc:3349-3381.
 * Two draws; sum = g1 + g2*2^32 (one rounding), / 2^64. */
static double rng_canonical(epo_rng* r) {
  double g1 = (double)rng_next(r);
  double g2 = (double)rng_next(r);
  double sum = g1 + g2 * 4294967296.0;
  double ret = sum / 18446744073709551616.0;
  if (ret >= 1.0) ret = nextafter(1.0, 0.0);
  return ret;
}

/* std::uniform_real_distribution<double>(a,b): bits/random.h operator():
 * (canonical * (b - a)) + a */
static double rng_uniform_real(epo_rng* r, double a, double b) {
  return rng_canonical(r) * (b - a) + a;
}

/* std::uniform_int_distribution<int>(a,b) on a 32-bit engine: Lemire's nearly
 * divisionless method, bits/uniform_int_dist.h:252-282,300-326. */
static int rng_uniform_int(epo_rng* r, int a, int b) {
  uint32_t range = (uint32_t)b - (uint32_t)a + 1u;
  uint64_t product = (uint64_t)rng_next(r) * (uint64_t)range;
  uint32_t low = (uint32_t)product;
  if (low < range) {
    uint32_t threshold = (0u - range) % range;
    while (low < threshold) {
      product = (uint64_t)rng_next(r) * (uint64_t)range;
      low = (uint32_t)product;
    }
  }
  return a + (int)(product >> 32);
}

/* std::normal_distribution<double>(mean, stddev): Marsaglia polar,
 * bits/random.tcc:1811-1844.  Returns y*mult first and caches x*mult. */
static double rng_normal(epo_rng* r, double mean, double stddev) {
  double ret;
  if (r->norm_has_saved) {
    r->norm_has_saved = 0;
    ret = r->norm_saved;
  } else {
    double x, y, r2;
    do {
      x = 2.0 * rng_canonical(r) - 1.0;
      y = 2.0 * rng_canonical(r) - 1.0;
      r2 = x * x + y * y;
    } while (r2 > 1.0 || r2 == 0.0);
    double mult = sqrt(-2 * log(r2) / r2);
    r->norm_saved = x * mult;
    r->norm_has_saved = 1;
    ret = y * mult;
  }
  return ret * stddev + mean;
}

/* callbacks handed to mjc_oracle.c (keeps that file free of the RNG layout) */
static double cb_uniform(void* ctx, double a, double b) {
  return rng_uniform_real((epo_rng*)ctx, a, b);
}
static double cb_normal(void* ctx, double mean, double stddev) {
  return rng_normal((epo_rng*)ctx, mean, stddev);
}

/* ------------------------------------------------------------- env state --- */
typedef struct {
  epo_rng rng;
  int done;         /* XxxEnv::done_, starts true (e.g. cartpole.h:67) */
  int current_step; /* Env::current_step_, starts -1 (core/env.h:81) */
  int elapsed;      /* XxxEnv::elapsed_step_ */
  double s[5];      /* continuous state */
  int i[8];         /* integer state */
  /* Blackjack hands (toy_text/blackjack.h:53) */
  int player[32], nplayer, dealer[32], ndealer;
  mjc_data* mj;     /* HalfCheetah only */
} epo_env;

#define EPO_MAX_KEYS 16
typedef struct {
  const char* name;
  int elem_size;
  int row_elems;
  void* data;
} epo_key;

struct epo_pool {
  int kind, num_envs, max_episode_steps, iopt;
  epo_env* envs;
  int nkeys;
  epo_key keys[EPO_MAX_KEYS];
  int act_elem_size, act_row_elems;
  mjc_model* mj_model;
  /* HalfCheetah's task options (half_cheetah.h:32-42, 84-95) */
  int hc_frame_skip;
  double hc_ctrl_cost_weight, hc_forward_reward_weight, hc_reset_noise_scale;
};

/* per-step result scratch */
typedef struct {
  float reward;
  float obs_f[64];
  int32_t obs_i[4];
  float extra_f[4];
  double obs_d[32];
  double info_d[4];
} epo_out;

/* ------------------------------------------------------- classic_control --- */
/* classic_control/cartpole.h:82-129 */
static void cartpole_write(const epo_env* e, epo_out* o, float reward) {
  for (int k = 0; k < 4; ++k) o->obs_f[k] = (float)e->s[k];
  o->reward = reward;
}
static void cartpole_reset(epo_env* e, epo_out* o) {
  for (int k = 0; k < 4; ++k) e->s[k] = rng_uniform_real(&e->rng, -0.05, 0.05);
  e->done = 0;
  e->elapsed = 0;
  cartpole_write(e, o, 0.0f);
}
static void cartpole_step(epo_env* e, int max_steps, int act, epo_out* o) {
  const double kGravity = 9.8, kMassCart = 1.0, kMassPole = 0.1;
  const double kMassTotal = kMassCart + kMassPole, kLength = 0.5;
  const double kMassPoleLength = kMassPole * kLength, kForceMag = 10.0;
  const double kTau = 0.02, kThetaThresholdRadians = 12 * 2 * M_PI / 360;
  const double kXThreshold = 2.4;
  double x = e->s[0], x_dot = e->s[1], theta = e->s[2], theta_dot = e->s[3];
  e->done = (++e->elapsed >= max_steps);
  double force = act == 1 ? kForceMag : -kForceMag;
  double costheta = cos(theta), sintheta = sin(theta);
  double temp =
      (force + kMassPoleLength * theta_dot * theta_dot * sintheta) / kMassTotal;
  double theta_acc =
      (kGravity * sintheta - costheta * temp) /
      (kLength * (4.0 / 3.0 - kMassPole * costheta * costheta / kMassTotal));
  double x_acc = temp - kMassPoleLength * theta_acc * costheta / kMassTotal;
  x += kTau * x_dot;
  x_dot += kTau * x_acc;
  theta += kTau * theta_dot;
  theta_dot += kTau * theta_acc;
  if (x < -kXThreshold || x > kXThreshold || theta < -kThetaThresholdRadians ||
      theta > kThetaThresholdRadians) {
    e->done = 1;
  }
  e->s[0] = x; e->s[1] = x_dot; e->s[2] = theta; e->s[3] = theta_dot;
  cartpole_write(e, o, 1.0f);
}

/* classic_control/pendulum.h:77-135 */
static void pendulum_write(const epo_env* e, epo_out* o, float reward) {
  o->obs_f[0] = (float)cos(e->s[0]);
  o->obs_f[1] = (float)sin(e->s[0]);
  o->obs_f[2] = (float)e->s[1];
  o->reward = reward;
}
static void pendulum_reset(epo_env* e, epo_out* o) {
  e->s[0] = rng_uniform_real(&e->rng, -M_PI, M_PI);
  e->s[1] = rng_uniform_real(&e->rng, -1, 1);
  e->done = 0;
  e->elapsed = 0;
  pendulum_write(e, o, 0.0f);
}
static void pendulum_step(epo_env* e, int max_steps, int version, float act,
                          epo_out* o) {
  const double kMaxSpeed = 8, kMaxTorque = 2, kDt = 0.05, kGravity = 10;
  double theta = e->s[0], theta_dot = e->s[1];
  e->done = (++e->elapsed >= max_steps);
  double u = act;
  if (act < -kMaxTorque) {
    u = -kMaxTorque;
  } else if (act > kMaxTorque) {
    u = kMaxTorque;
  }
  double cost = theta * theta + 0.1 * theta_dot * theta_dot + 0.001 * u * u;
  double new_theta_dot = theta_dot + 3 * (kGravity / 2 * sin(theta) + u) * kDt;
  if (version == 0) theta += new_theta_dot * kDt;
  theta_dot = new_theta_dot;
  if (new_theta_dot < -kMaxSpeed) {
    theta_dot = -kMaxSpeed;
  } else if (new_theta_dot > kMaxSpeed) {
    theta_dot = kMaxSpeed;
  }
  if (version == 1) theta += new_theta_dot * kDt;
  while (theta < -M_PI) theta += M_PI * 2;
  while (theta >= M_PI) theta -= M_PI * 2;
  e->s[0] = theta; e->s[1] = theta_dot;
  pendulum_write(e, o, (float)(-cost));
}

/* classic_control/acrobot.h:94-191 */
typedef struct { double s0, s1, s2, s3, s4; } v5;
static v5 v5_add(v5 a, v5 b) {
  v5 r = {a.s0 + b.s0, a.s1 + b.s1, a.s2 + b.s2, a.s3 + b.s3, a.s4 + b.s4};
  return r;
}
static v5 v5_mul(v5 a, double v) {
  v5 r = {a.s0 * v, a.s1 * v, a.s2 * v, a.s3 * v, a.s4 * v};
  return r;
}
static v5 acrobot_derivs(v5 s) { /* acrobot.h:158-178 */
  const double kG = 9.8, kL = 1.0, kM = 1.0, kLC = 0.5, kI = 1.0;
  double theta1 = s.s0, theta2 = s.s1, dtheta1 = s.s2, dtheta2 = s.s3, a = s.s4;
  double d1 = kM * kLC * kLC +
              kM * (kL * kL + kLC * kLC + 2 * kL * kLC * cos(theta2)) + kI * 2;
  double d2 = kM * (kLC * kLC + kL * kLC * cos(theta2)) + kI;
  double phi2 = kM * kLC * kG * cos(theta1 + theta2 - M_PI / 2);
  double phi1 =
      -(dtheta2 + 2 * dtheta1) * kM * kL * kLC * dtheta2 * sin(theta2) +
      kM * (kLC + kL) * kG * cos(theta1 - M_PI / 2) + phi2;
  double ddtheta2 = (a + d2 / d1 * phi1 -
                     kM * kL * kLC * dtheta1 * dtheta1 * sin(theta2) - phi2) /
                    (kM * kLC * kLC + kI - d2 * d2 / d1);
  double ddtheta1 = -(d2 * ddtheta2 + phi1) / d1;
  v5 r = {dtheta1, dtheta2, ddtheta1, ddtheta2, 0};
  return r;
}
static v5 acrobot_rk4(v5 y0) { /* acrobot.h:150-156 */
  const double kDt = 0.2;
  v5 k1 = acrobot_derivs(y0);
  v5 k2 = acrobot_derivs(v5_add(y0, v5_mul(k1, kDt / 2)));
  v5 k3 = acrobot_derivs(v5_add(y0, v5_mul(k2, kDt / 2)));
  v5 k4 = acrobot_derivs(v5_add(y0, v5_mul(k3, kDt)));
  v5 sum = v5_add(v5_add(v5_add(k1, v5_mul(k2, 2)), v5_mul(k3, 2)), k4);
  return v5_add(y0, v5_mul(sum, kDt / 6.0));
}
static void acrobot_write(const epo_env* e, epo_out* o, float reward) {
  o->obs_f[0] = (float)cos(e->s[0]);
  o->obs_f[1] = (float)sin(e->s[0]);
  o->obs_f[2] = (float)cos(e->s[1]);
  o->obs_f[3] = (float)sin(e->s[1]);
  o->obs_f[4] = (float)e->s[2];
  o->obs_f[5] = (float)e->s[3];
  o->extra_f[0] = (float)e->s[0];
  o->extra_f[1] = (float)e->s[1];
  o->reward = reward;
}
static void acrobot_reset(epo_env* e, epo_out* o) {
  for (int k = 0; k < 4; ++k) e->s[k] = rng_uniform_real(&e->rng, -0.1, 0.1);
  e->s[4] = 0;
  e->done = 0;
  e->elapsed = 0;
  acrobot_write(e, o, 0.0f);
}
static void acrobot_step(epo_env* e, int max_steps, int act, epo_out* o) {
  const double kMaxVel1 = 4 * M_PI, kMaxVel2 = 9 * M_PI;
  e->done = (++e->elapsed >= max_steps);
  float reward = -1.0f;
  v5 s = {e->s[0], e->s[1], e->s[2], e->s[3], (double)(act - 1)};
  s = acrobot_rk4(s);
  while (s.s0 < -M_PI) s.s0 += M_PI * 2;
  while (s.s1 < -M_PI) s.s1 += M_PI * 2;
  while (s.s0 >= M_PI) s.s0 -= M_PI * 2;
  while (s.s1 >= M_PI) s.s1 -= M_PI * 2;
  if (s.s2 < -kMaxVel1) s.s2 = -kMaxVel1;
  if (s.s3 < -kMaxVel2) s.s3 = -kMaxVel2;
  if (s.s2 > kMaxVel1) s.s2 = kMaxVel1;
  if (s.s3 > kMaxVel2) s.s3 = kMaxVel2;
  if (-cos(s.s0) - cos(s.s0 + s.s1) > 1) {
    e->done = 1;
    reward = 0.0f;
  }
  e->s[0] = s.s0; e->s[1] = s.s1; e->s[2] = s.s2; e->s[3] = s.s3; e->s[4] = s.s4;
  acrobot_write(e, o, reward);
}

/* classic_control/mountain_car.h:76-119, mountain_car_continuous.h:77-127 */
static void mcar_write(const epo_env* e, epo_out* o, float reward) {
  o->obs_f[0] = (float)e->s[0];
  o->obs_f[1] = (float)e->s[1];
  o->reward = reward;
}
static void mcar_reset(epo_env* e, epo_out* o) {
  e->s[0] = rng_uniform_real(&e->rng, -0.6, -0.4);
  e->s[1] = 0.0;
  e->done = 0;
  e->elapsed = 0;
  mcar_write(e, o, 0.0f);
}
static void mcar_common(epo_env* e, double accel, double goal_pos) {
  const double kMinPos = -1.2, kMaxPos = 0.6, kMaxSpeed = 0.07;
  const double kGoalVel = 0, kGravity = 0.0025;
  double pos = e->s[0], vel = e->s[1];
  vel += accel - cos(3 * pos) * kGravity;
  if (vel < -kMaxSpeed) {
    vel = -kMaxSpeed;
  } else if (vel > kMaxSpeed) {
    vel = kMaxSpeed;
  }
  pos += vel;
  if (pos < kMinPos) {
    pos = kMinPos;
  } else if (pos > kMaxPos) {
    pos = kMaxPos;
  }
  if (pos == kMinPos && vel < 0) vel = 0;
  e->s[0] = pos; e->s[1] = vel;
  e->i[0] = (pos >= goal_pos && vel >= kGoalVel);
}
static void mcar_step(epo_env* e, int max_steps, int action, epo_out* o) {
  e->done = (++e->elapsed >= max_steps);
  double act = action - 1;
  mcar_common(e, act * 0.001, 0.5);
  if (e->i[0]) e->done = 1;
  mcar_write(e, o, -1.0f);
}
static void mcarc_step(epo_env* e, int max_steps, float action, epo_out* o) {
  e->done = (++e->elapsed >= max_steps);
  double act = action;
  double reward = -0.1 * act * act;
  if (act < -1) {
    act = -1;
  } else if (act > 1) {
    act = 1;
  }
  mcar_common(e, act * 0.0015, 0.45);
  if (e->i[0]) {
    e->done = 1;
    reward += 100;
  }
  mcar_write(e, o, (float)reward);
}

/* -------------------------------------------------------------- toy_text --- */
/* toy_text/frozen_lake.h:58-108 ; i[0]=x_, i[1]=y_ */
static const char* kLake4[4] = {"SFFF", "FHFH", "FFFH", "HFFG"};
static const char* kLake8[8] = {"SFFFFFFF", "FFFFFFFF", "FFFHFFFF", "FFFFFHFF",
                                "FFFHFFFF", "FHHFFFHF", "FHFFHFHF", "FFFHFFFG"};
static void lake_reset(epo_env* e, int size, epo_out* o) {
  e->i[0] = e->i[1] = 0;
  e->done = 0;
  e->elapsed = 0;
  o->obs_i[0] = e->i[0] * size + e->i[1];
  o->reward = 0.0f;
}
static void lake_step(epo_env* e, int max_steps, int size, int act, epo_out* o) {
  const char** map = size != 8 ? kLake4 : kLake8;
  int x = e->i[0], y = e->i[1];
  e->done = (++e->elapsed >= max_steps);
  act = (act + rng_uniform_int(&e->rng, -1, 1) + 4) % 4;
  if (act == 0) {
    --y;
  } else if (act == 1) {
    ++x;
  } else if (act == 2) {
    ++y;
  } else {
    --x;
  }
  x = x < 0 ? 0 : (x > size - 1 ? size - 1 : x);
  y = y < 0 ? 0 : (y > size - 1 ? size - 1 : y);
  float reward = 0.0f;
  if (map[x][y] == 'H' || map[x][y] == 'G') {
    e->done = 1;
    reward = map[x][y] == 'G' ? 1.0f : 0.0f;
  }
  e->i[0] = x; e->i[1] = y;
  o->obs_i[0] = x * size + y;
  o->reward = reward;
}

/* toy_text/catch.h:62-93 ; i[0]=x_, i[1]=y_, i[2]=paddle_.  The output grid is
 * zero-filled because a fresh StateBuffer is used per Recv (state_buffer_queue.h). */
static void catch_write(const epo_env* e, epo_out* o, float reward) {
  memset(o->obs_f, 0, sizeof(float) * 50);
  o->obs_f[e->i[0] * 5 + e->i[1]] = 1.0f;
  o->obs_f[9 * 5 + e->i[2]] = 1.0f;
  o->reward = reward;
}
static void catch_reset(epo_env* e, epo_out* o) {
  e->i[0] = 0;
  e->i[1] = rng_uniform_int(&e->rng, 0, 4);
  e->i[2] = 5 / 2;
  e->done = 0;
  catch_write(e, o, 0.0f);
}
static void catch_step(epo_env* e, int act, epo_out* o) {
  float reward = 0.0f;
  e->i[2] += act - 1;
  if (e->i[2] < 0) e->i[2] = 0;
  if (e->i[2] >= 5) e->i[2] = 4;
  if (++e->i[0] == 10 - 1) {
    e->done = 1;
    reward = e->i[1] == e->i[2] ? 1.0f : -1.0f;
  }
  catch_write(e, o, reward);
}

/* toy_text/taxi.h:69-127 ; i[0]=x_, i[1]=y_, i[2]=s_, i[3]=t_ */
static const int kTaxiLoc[4][2] = {{0, 0}, {0, 4}, {4, 0}, {4, 3}};
static const char* kTaxiMap[5] = {"|:|::|", "|:|::|", "|::::|", "||:|:|", "||:|:|"};
static const char* kTaxiLocMap[5] = {"0   1", "     ", "     ", "     ", "2  3 "};
static void taxi_write(const epo_env* e, epo_out* o, float reward) {
  o->obs_i[0] = ((e->i[0] * 5 + e->i[1]) * 5 + e->i[2]) * 4 + e->i[3];
  o->reward = reward;
}
static void taxi_reset(epo_env* e, epo_out* o) {
  e->i[0] = rng_uniform_int(&e->rng, 0, 4);
  e->i[1] = rng_uniform_int(&e->rng, 0, 4);
  e->i[2] = rng_uniform_int(&e->rng, 0, 3);
  e->i[3] = rng_uniform_int(&e->rng, 0, 3);
  e->done = 0;
  e->elapsed = 0;
  taxi_write(e, o, 0.0f);
}
static void taxi_step(epo_env* e, int max_steps, int act, epo_out* o) {
  int x = e->i[0], y = e->i[1], s = e->i[2], t = e->i[3];
  e->done = (++e->elapsed >= max_steps);
  float reward = -1.0f;
  if (act == 0) {
    if (x < 4) ++x;
  } else if (act == 1) {
    if (x > 0) --x;
  } else if (act == 2) {
    if (kTaxiMap[x][y + 1] == ':') ++y;
  } else if (act == 3) {
    if (kTaxiMap[x][y] == ':') --y;
  } else if (act == 4) {
    if (s < 4 && x == kTaxiLoc[s][0] && y == kTaxiLoc[s][1]) {
      s = 4;
    } else {
      reward = -10.0f;
    }
  } else {
    if (s == 4 && x == kTaxiLoc[t][0] && y == kTaxiLoc[t][1]) {
      s = t;
      e->done = 1;
      reward = 20.0f;
    } else if (s == 4 && kTaxiLocMap[x][y] != ' ') {
      s = kTaxiLocMap[x][y] - '0';
    } else {
      reward = -10.0f;
    }
  }
  e->i[0] = x; e->i[1] = y; e->i[2] = s; e->i[3] = t;
  taxi_write(e, o, reward);
}

/* toy_text/nchain.h:61-92 ; i[0]=s_ */
static void nchain_reset(epo_env* e, epo_out* o) {
  e->i[0] = 0;
  e->done = 0;
  e->elapsed = 0;
  o->obs_i[0] = 0;
  o->reward = 0.0f;
}
static void nchain_step(epo_env* e, int max_steps, int act, epo_out* o) {
  e->done = (++e->elapsed >= max_steps);
  if (rng_uniform_real(&e->rng, 0, 1) < 0.2) act = 1 - act;
  float reward = 0.0f;
  if (act != 0) {
    reward = 2.0f;
    e->i[0] = 0;
  } else if (e->i[0] < 4) {
    ++e->i[0];
  } else {
    reward = 10.0f;
  }
  o->obs_i[0] = e->i[0];
  o->reward = reward;
}

/* toy_text/cliffwalking.h:64-111 ; i[0]=x_, i[1]=y_ */
static void cliff_write(const epo_env* e, epo_out* o, float reward, float prob) {
  o->obs_i[0] = e->i[0] * 12 + e->i[1];
  o->reward = reward;
  o->extra_f[0] = prob;
}
static void cliff_reset(epo_env* e, epo_out* o) {
  e->i[0] = 3;
  e->i[1] = 0;
  e->done = 0;
  cliff_write(e, o, 0.0f, 1.0f);
}
static void cliff_step(epo_env* e, int slippery, int act, epo_out* o) {
  if (slippery) {
    static const int k_offsets[3] = {-1, 0, 1};
    act = (act + k_offsets[rng_uniform_int(&e->rng, 0, 2)] + 4) % 4;
  }
  int x = e->i[0], y = e->i[1];
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
  x = x > 0 ? x : 0; x = x < 3 ? x : 3;
  y = y > 0 ? y : 0; y = y < 11 ? y : 11;
  if (x == 3 && y > 0 && y < 11) {
    reward = -100.0f;
    x = 3;
    y = 0;
  }
  if (x == 3 && y == 11) e->done = 1;
  e->i[0] = x; e->i[1] = y;
  cliff_write(e, o, reward, slippery ? 1.0f / 3.0f : 1.0f);
}

/* toy_text/blackjack.h:65-147 */
static int bj_draw(epo_env* e) {
  int c = rng_uniform_int(&e->rng, 1, 13);
  return c < 10 ? c : 10;
}
static int bj_usable_ace(const int* h, int n) {
  for (int k = 0; k < n; ++k)
    if (h[k] == 1) return 1;
  return 0;
}
static int bj_sum(const int* h, int n) {
  int sum = 0;
  for (int k = 0; k < n; ++k) sum += h[k];
  if (bj_usable_ace(h, n) != 0 && sum + 10 <= 21) return sum + 10;
  return sum;
}
static int bj_score(const int* h, int n) {
  int r = bj_sum(h, n);
  return r > 21 ? 0 : r;
}
static int bj_natural(const int* h, int n) {
  return n == 2 && ((h[0] == 1 && h[1] == 10) || (h[0] == 10 && h[1] == 1));
}
static void bj_write(const epo_env* e, epo_out* o, float reward) {
  o->obs_i[0] = bj_sum(e->player, e->nplayer);
  o->obs_i[1] = e->dealer[0];
  o->obs_i[2] = bj_usable_ace(e->player, e->nplayer);
  o->reward = reward;
}
static void bj_reset(epo_env* e, epo_out* o) {
  e->nplayer = 0;
  e->player[e->nplayer++] = bj_draw(e);
  e->player[e->nplayer++] = bj_draw(e);
  e->ndealer = 0;
  e->dealer[e->ndealer++] = bj_draw(e);
  e->dealer[e->ndealer++] = bj_draw(e);
  e->done = 0;
  bj_write(e, o, 0.0f);
}
static void bj_step(epo_env* e, int natural, int sab, int act, epo_out* o) {
  float reward = 0.0f;
  if (act != 0) {
    e->player[e->nplayer++] = bj_draw(e);
    if (bj_sum(e->player, e->nplayer) > 21) {
      e->done = 1;
      reward = -1.0f;
    }
  } else {
    e->done = 1;
    while (bj_sum(e->dealer, e->ndealer) < 17) e->dealer[e->ndealer++] = bj_draw(e);
    int ps = bj_score(e->player, e->nplayer);
    int ds = bj_score(e->dealer, e->ndealer);
    reward = (ps > ds ? 1.0f : 0.0f) - (ps < ds ? 1.0f : 0.0f);
    if (sab && bj_natural(e->player, e->nplayer) &&
        !bj_natural(e->dealer, e->ndealer)) {
      reward = 1.0f;
    } else if (!sab && natural && bj_natural(e->player, e->nplayer) &&
               reward == 1.0f) {
      reward = 1.5f;
    }
  }
  bj_write(e, o, reward);
}

/* ------------------------------------------------------------------ pool --- */
static void add_key(epo_pool* p, const char* name, int elem, int row) {
  epo_key* k = &p->keys[p->nkeys++];
  k->name = name;
  k->elem_size = elem;
  k->row_elems = row;
  k->data = calloc((size_t)p->num_envs * row, elem);
}

epo_pool* epo_create(int kind, int num_envs, int seed, const int* env_seed,
                     int max_episode_steps, int iopt, int frame_skip, double ctrl_cost_weight,
                     double forward_reward_weight, double reset_noise_scale) {
  if (kind < 0 || kind >= EPO_NUM_KINDS || num_envs <= 0) return NULL;
  epo_pool* p = (epo_pool*)calloc(1, sizeof(epo_pool));
  p->hc_frame_skip = frame_skip;
  p->hc_ctrl_cost_weight = ctrl_cost_weight;
  p->hc_forward_reward_weight = forward_reward_weight;
  p->hc_reset_noise_scale = reset_noise_scale;
  p->kind = kind;
  p->num_envs = num_envs;
  p->max_episode_steps = max_episode_steps > 0 ? max_episode_steps : INT_MAX;
  p->iopt = iopt;
  if (iopt < 0) { /* reference defaults */
    p->iopt = kind == EPO_FROZEN_LAKE ? 4 : kind == EPO_BLACKJACK ? 2 : 0;
  }
  /* common state keys, order of core/env_spec.h:37-43 */
  add_key(p, "info:env_id", 4, 1);
  add_key(p, "info:players.env_id", 4, 1);
  add_key(p, "elapsed_step", 4, 1);
  add_key(p, "done", 1, 1);
  add_key(p, "reward", 4, 1);
  add_key(p, "discount", 4, 1);
  add_key(p, "step_type", 4, 1);
  add_key(p, "trunc", 1, 1);
  p->act_elem_size = 4;
  p->act_row_elems = 1;
  switch (kind) {
    case EPO_CARTPOLE: add_key(p, "obs", 4, 4); break;
    case EPO_PENDULUM: add_key(p, "obs", 4, 3); break;
    case EPO_ACROBOT: add_key(p, "obs", 4, 6); add_key(p, "info:state", 4, 2); break;
    case EPO_MOUNTAIN_CAR:
    case EPO_MOUNTAIN_CAR_CONTINUOUS: add_key(p, "obs", 4, 2); break;
    case EPO_FROZEN_LAKE: case EPO_TAXI: case EPO_NCHAIN: add_key(p, "obs", 4, 1); break;
    case EPO_CATCH: add_key(p, "obs", 4, 50); break;
    case EPO_CLIFF_WALKING: add_key(p, "obs", 4, 1); add_key(p, "info:prob", 4, 1); break;
    case EPO_BLACKJACK: add_key(p, "obs", 4, 3); break;
    case EPO_HALF_CHEETAH:
      /* mujoco/gym/half_cheetah.h:44-62 (non-test build: no qpos0/qvel0 keys) */
      add_key(p, "obs", 8, 17);
      add_key(p, "info:reward_run", 8, 1);
      add_key(p, "info:reward_ctrl", 8, 1);
      add_key(p, "info:x_position", 8, 1);
      add_key(p, "info:x_velocity", 8, 1);
      p->act_elem_size = 8;
      p->act_row_elems = 6;
      p->mj_model = mjc_make_half_cheetah();
      break;
  }
  p->envs = (epo_env*)calloc((size_t)num_envs, sizeof(epo_env));
  for (int e = 0; e < num_envs; ++e) {
    /* Env::ResolveSeed, core/env.h:101-111 */
    int s = env_seed ? env_seed[e] : seed + e;
    rng_seed(&p->envs[e].rng, (uint32_t)s);
    p->envs[e].done = 1;
    p->envs[e].current_step = -1;
    p->envs[e].elapsed = p->max_episode_steps + 1; /* unused before first reset */
    if (kind == EPO_HALF_CHEETAH) p->envs[e].mj = mjc_make_data(p->mj_model);
  }
  return p;
}

void epo_destroy(epo_pool* p) {
  if (!p) return;
  for (int k = 0; k < p->nkeys; ++k) free(p->keys[k].data);
  if (p->kind == EPO_HALF_CHEETAH) {
    for (int e = 0; e < p->num_envs; ++e) mjc_free_data(p->envs[e].mj);
    mjc_free_model(p->mj_model);
  }
  free(p->envs);
  free(p);
}

/* Env::EnvStep + Env::Allocate for one env, writing output row `row`
 * (core/env.h:184-256; worker loop core/async_envpool.h:118-131). */
static void env_step_row(epo_pool* p, int eid, int row, const void* action,
                         int force_reset) {
  epo_env* e = &p->envs[eid];
  epo_out o;
  memset(&o, 0, sizeof(o));
  int reset = force_reset || e->done; /* async_envpool.h:127 */
  if (reset) {
    e->current_step = 0; /* PreProcess, env.h:207-217 */
  } else {
    ++e->current_step;
  }
  const int32_t* ai = (const int32_t*)action;
  const float* af = (const float*)action;
  int ms = p->max_episode_steps;
  switch (p->kind) {
    case EPO_CARTPOLE:
      if (reset) cartpole_reset(e, &o); else cartpole_step(e, ms, ai[row], &o);
      break;
    case EPO_PENDULUM:
      if (reset) pendulum_reset(e, &o); else pendulum_step(e, ms, p->iopt, af[row], &o);
      break;
    case EPO_ACROBOT:
      if (reset) acrobot_reset(e, &o); else acrobot_step(e, ms, ai[row], &o);
      break;
    case EPO_MOUNTAIN_CAR:
      if (reset) mcar_reset(e, &o); else mcar_step(e, ms, ai[row], &o);
      break;
    case EPO_MOUNTAIN_CAR_CONTINUOUS:
      if (reset) mcar_reset(e, &o); else mcarc_step(e, ms, af[row], &o);
      break;
    case EPO_FROZEN_LAKE:
      if (reset) lake_reset(e, p->iopt, &o); else lake_step(e, ms, p->iopt, ai[row], &o);
      break;
    case EPO_CATCH:
      if (reset) catch_reset(e, &o); else catch_step(e, ai[row], &o);
      break;
    case EPO_TAXI:
      if (reset) taxi_reset(e, &o); else taxi_step(e, ms, ai[row], &o);
      break;
    case EPO_NCHAIN:
      if (reset) nchain_reset(e, &o); else nchain_step(e, ms, ai[row], &o);
      break;
    case EPO_CLIFF_WALKING:
      if (reset) cliff_reset(e, &o); else cliff_step(e, p->iopt, ai[row], &o);
      break;
    case EPO_BLACKJACK:
      if (reset) bj_reset(e, &o); else bj_step(e, p->iopt & 1, (p->iopt >> 1) & 1, ai[row], &o);
      break;
    case EPO_HALF_CHEETAH: {
      /* mujoco/gym/half_cheetah.h:127-156 and WriteState, :164-185 */
      const double fwd = p->hc_forward_reward_weight;
      if (reset) {
        e->done = 0;
        e->elapsed = 0;
        mjc_reset(p->mj_model, e->mj, p->hc_reset_noise_scale, cb_uniform, cb_normal, &e->rng);
        o.reward = 0.0f;
        /* WriteState(0.0, 0.0, 0.0, 0.0, true): reward_run = 0.0 * fwd (-0.0 when fwd < 0) */
        o.info_d[0] = 0.0 * fwd; o.info_d[1] = -0.0; o.info_d[2] = 0.0; o.info_d[3] = 0.0;
      } else {
        const double* act = (const double*)action + (size_t)row * 6;
        double x_before = mjc_qpos(e->mj)[0];
        mjc_step(p->mj_model, e->mj, act, p->hc_frame_skip);
        double x_after = mjc_qpos(e->mj)[0];
        double ctrl_cost = 0.0;
        for (int k = 0; k < 6; ++k) ctrl_cost += p->hc_ctrl_cost_weight * act[k] * act[k];
        double dt = p->hc_frame_skip * 0.01;
        double xv = (x_after - x_before) / dt;
        o.reward = (float)(xv * fwd - ctrl_cost);
        e->done = (++e->elapsed >= ms);
        o.info_d[0] = xv * fwd; o.info_d[1] = -ctrl_cost;
        o.info_d[2] = x_after; o.info_d[3] = xv;
      }
      const double* qpos = mjc_qpos(e->mj);
      const double* qvel = mjc_qvel(e->mj);
      for (int k = 1; k < 9; ++k) o.obs_d[k - 1] = qpos[k];
      for (int k = 0; k < 9; ++k) o.obs_d[8 + k] = qvel[k];
      break;
    }
  }
  /* Env::Allocate common columns, core/env.h:224-256 */
  int done = e->done;
  int step_type = 1;
  if (e->current_step == 0) {
    step_type = 0;
  } else if (done) {
    step_type = 2;
  }
  ((int32_t*)p->keys[0].data)[row] = eid;
  ((int32_t*)p->keys[1].data)[row] = eid;
  ((int32_t*)p->keys[2].data)[row] = e->current_step;
  ((uint8_t*)p->keys[3].data)[row] = (uint8_t)done;
  ((float*)p->keys[4].data)[row] = o.reward;
  ((float*)p->keys[5].data)[row] = (float)(!done);
  ((int32_t*)p->keys[6].data)[row] = step_type;
  ((uint8_t*)p->keys[7].data)[row] =
      (uint8_t)(done && (e->current_step >= p->max_episode_steps));
  /* env-specific columns */
  epo_key* k8 = &p->keys[8];
  switch (p->kind) {
    case EPO_CARTPOLE: case EPO_PENDULUM: case EPO_MOUNTAIN_CAR:
    case EPO_MOUNTAIN_CAR_CONTINUOUS: case EPO_CATCH:
      memcpy((float*)k8->data + (size_t)row * k8->row_elems, o.obs_f,
             sizeof(float) * k8->row_elems);
      break;
    case EPO_ACROBOT:
      memcpy((float*)k8->data + (size_t)row * 6, o.obs_f, sizeof(float) * 6);
      memcpy((float*)p->keys[9].data + (size_t)row * 2, o.extra_f, sizeof(float) * 2);
      break;
    case EPO_FROZEN_LAKE: case EPO_TAXI: case EPO_NCHAIN:
      ((int32_t*)k8->data)[row] = o.obs_i[0];
      break;
    case EPO_CLIFF_WALKING:
      ((int32_t*)k8->data)[row] = o.obs_i[0];
      ((float*)p->keys[9].data)[row] = o.extra_f[0];
      break;
    case EPO_BLACKJACK:
      memcpy((int32_t*)k8->data + (size_t)row * 3, o.obs_i, sizeof(int32_t) * 3);
      break;
    case EPO_HALF_CHEETAH:
      memcpy((double*)k8->data + (size_t)row * 17, o.obs_d, sizeof(double) * 17);
      for (int k = 0; k < 4; ++k) ((double*)p->keys[9 + k].data)[row] = o.info_d[k];
      break;
  }
}

void epo_reset(epo_pool* p, const int32_t* env_ids, int n) {
  for (int i = 0; i < n; ++i) env_step_row(p, env_ids ? env_ids[i] : i, i, NULL, 1);
}

void epo_step(epo_pool* p, const void* action, const int32_t* env_ids, int n) {
  for (int i = 0; i < n; ++i) env_step_row(p, env_ids ? env_ids[i] : i, i, action, 0);
}

int epo_num_keys(const epo_pool* p) { return p->nkeys; }
const char* epo_key_name(const epo_pool* p, int k) { return p->keys[k].name; }
int epo_key_elem_size(const epo_pool* p, int k) { return p->keys[k].elem_size; }
int epo_key_row_elems(const epo_pool* p, int k) { return p->keys[k].row_elems; }
const void* epo_key_data(const epo_pool* p, int k) { return p->keys[k].data; }
int epo_action_elem_size(const epo_pool* p) { return p->act_elem_size; }
int epo_action_row_elems(const epo_pool* p) { return p->act_row_elems; }
void epo_get_state(const epo_pool* p, int eid, double* s5, int* done, int* cur) {
  const epo_env* e = &p->envs[eid];
  for (int k = 0; k < 5; ++k) s5[k] = e->s[k];
  *done = e->done;
  *cur = e->current_step;
}
void epo_get_states(const epo_pool* p, double* s5) {
  for (int e = 0; e < p->num_envs; ++e) memcpy(s5 + (size_t)e * 5, p->envs[e].s, sizeof(double) * 5);
}
void epo_set_state(epo_pool* p, int eid, const double* s5, int done, int cur) {
  epo_env* e = &p->envs[eid];
  for (int k = 0; k < 5; ++k) e->s[k] = s5[k];
  e->done = done;
  e->current_step = cur;
  e->elapsed = cur;
}
void epo_set_int_states(epo_pool* p, const int32_t* i8, const int32_t* player32,
                        const int32_t* nplayer, const int32_t* dealer32, const int32_t* ndealer,
                        const int32_t* done, const int32_t* cur) {
  for (int eid = 0; eid < p->num_envs; ++eid) {
    epo_env* e = &p->envs[eid];
    for (int k = 0; k < 8; ++k) e->i[k] = i8[(size_t)eid * 8 + k];
    if (player32) {
      e->nplayer = nplayer[eid];
      e->ndealer = ndealer[eid];
      for (int k = 0; k < 32; ++k) {
        e->player[k] = player32[(size_t)eid * 32 + k];
        e->dealer[k] = dealer32[(size_t)eid * 32 + k];
      }
    }
    e->done = done[eid];
    e->current_step = cur[eid];
    e->elapsed = cur[eid];
  }
}
void epo_get_int_states(const epo_pool* p, int32_t* i8, int32_t* player32, int32_t* nplayer,
                        int32_t* dealer32, int32_t* ndealer, int32_t* done, int32_t* cur) {
  for (int eid = 0; eid < p->num_envs; ++eid) {
    const epo_env* e = &p->envs[eid];
    for (int k = 0; k < 8; ++k) i8[(size_t)eid * 8 + k] = e->i[k];
    if (player32) {
      nplayer[eid] = e->nplayer;
      ndealer[eid] = e->ndealer;
      for (int k = 0; k < 32; ++k) {
        player32[(size_t)eid * 32 + k] = e->player[k];
        dealer32[(size_t)eid * 32 + k] = e->dealer[k];
      }
    }
    done[eid] = e->done;
    cur[eid] = e->current_step;
  }
}
void epo_mjc_set(epo_pool* p, int eid, const double* s27, int done, int cur) {
  epo_env* e = &p->envs[eid];
  memcpy(mjc_qpos_mut(e->mj), s27, sizeof(double) * 9);
  memcpy(mjc_qvel_mut(e->mj), s27 + 9, sizeof(double) * 9);
  memcpy(mjc_warm_mut(e->mj), s27 + 18, sizeof(double) * 9);
  e->done = done;
  e->current_step = cur;
  e->elapsed = cur;
}
void epo_mjc_get(const epo_pool* p, int eid, double* s27) {
  const epo_env* e = &p->envs[eid];
  memcpy(s27, mjc_qpos(e->mj), sizeof(double) * 9);
  memcpy(s27 + 9, mjc_qvel(e->mj), sizeof(double) * 9);
  memcpy(s27 + 18, mjc_warm_mut(e->mj), sizeof(double) * 9);
}
uint32_t epo_debug_draw(epo_pool* p, int eid) { return rng_next(&p->envs[eid].rng); }
/* RNG recipe hooks for tests/test_oracle_rng_vs_libstdcxx.py: load an engine state
 * (624 words + read position, the representation std::mt19937's operator<< prints) and
 * call the restated distributions directly. */
void epo_debug_set_rng(epo_pool* p, int eid, const uint32_t* mt624, int idx) {
  epo_rng* r = &p->envs[eid].rng;
  memcpy(r->mt, mt624, sizeof(r->mt));
  r->idx = idx;
  r->norm_has_saved = 0;
  r->norm_saved = 0.0;
}
void epo_debug_get_rng(const epo_pool* p, int eid, uint32_t* mt624, int* idx) {
  const epo_rng* r = &p->envs[eid].rng;
  memcpy(mt624, r->mt, sizeof(r->mt));
  *idx = r->idx;
}
int epo_debug_uniform_int(epo_pool* p, int eid, int a, int b) {
  return rng_uniform_int(&p->envs[eid].rng, a, b);
}
double epo_debug_uniform_real(epo_pool* p, int eid, double a, double b) {
  return rng_uniform_real(&p->envs[eid].rng, a, b);
}
double epo_debug_normal(epo_pool* p, int eid, double mean, double stddev) {
  return rng_normal(&p->envs[eid].rng, mean, stddev);
}
int epo_trig(int kind, const void* x, int n, void* s, void* c) {
  if (kind == 0) {
    const double* xd = (const double*)x;
    for (int i = 0; i < n; ++i) {
      if (s) ((double*)s)[i] = sin(xd[i]);
      if (c) ((double*)c)[i] = cos(xd[i]);
    }
    return 0;
  }
  if (kind == 1) {
    const float* xf = (const float*)x;
    for (int i = 0; i < n; ++i) {
      if (s) ((float*)s)[i] = sinf(xf[i]);
      if (c) ((float*)c)[i] = cosf(xf[i]);
    }
    return 0;
  }
  return -1;
}
