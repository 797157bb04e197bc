/* TEST INFRASTRUCTURE ONLY -- CPU restatement ("oracle") of the reference hot path.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/reference legs may
 * load this.  The product (envpool_b200/) never links, imports or calls it.
 *
 * Parity status: PINNED for classic_control + toy_text -- checked bit-for-bit against
 * the reference itself compiled here (oracle/_ref, see oracle/Makefile) and against
 * the committed fixtures in tests/golden/ generated from it.
 * HalfCheetah (mjc_oracle.c): PARITY UNPINNED -- MuJoCo 3.6.0 is absent (see that
 * file's header).
 */
#ifndef EP_ORACLE_H_
#define EP_ORACLE_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum epo_kind {
  EPO_CARTPOLE = 0,
  EPO_PENDULUM = 1,
  EPO_ACROBOT = 2,
  EPO_MOUNTAIN_CAR = 3,
  EPO_MOUNTAIN_CAR_CONTINUOUS = 4,
  EPO_FROZEN_LAKE = 5,
  EPO_CATCH = 6,
  EPO_TAXI = 7,
  EPO_NCHAIN = 8,
  EPO_CLIFF_WALKING = 9,
  EPO_BLACKJACK = 10,
  EPO_HALF_CHEETAH = 11,
  EPO_NUM_KINDS = 12
};

typedef struct epo_pool epo_pool;

/* iopt: FrozenLake size / Pendulum version / CliffWalking is_slippery /
 * Blackjack (natural | sab<<1); -1 = reference default.
 * env_seed: optional per-env seeds (envpool/core/env.h:101-111), else seed+env_id.
 * max_episode_steps <= 0 selects INT_MAX (envpool/core/env_spec.h:31).
 * frame_skip, ctrl_cost_weight, forward_reward_weight, reset_noise_scale: HalfCheetah's task
 * options (mujoco/gym/half_cheetah.h:32-42), used as given (reference defaults 5, 0.1, 1.0,
 * 0.1); ignored by every other kind. */
epo_pool* epo_create(int kind, int num_envs, int seed, const int* env_seed,
                     int max_episode_steps, int iopt, int frame_skip, double ctrl_cost_weight,
                     double forward_reward_weight, double reset_noise_scale);
void epo_destroy(epo_pool* p);
/* Forced reset of the listed envs (AsyncEnvPool::Reset, async_envpool.h:224-237);
 * env_ids NULL = all envs in order.  Output row i <-> env_ids[i]. */
void epo_reset(epo_pool* p, const int32_t* env_ids, int n);
/* One Send+Recv in sync mode (async_envpool.h:59-82,118-131,169-181). */
void epo_step(epo_pool* p, const void* action, const int32_t* env_ids, int n);
int epo_num_keys(const epo_pool* p);
const char* epo_key_name(const epo_pool* p, int k);
/* element size in bytes and per-row element count of state key k */
int epo_key_elem_size(const epo_pool* p, int k);
int epo_key_row_elems(const epo_pool* p, int k);
/* data of state key k for the rows of the last reset/step call */
const void* epo_key_data(const epo_pool* p, int k);
int epo_action_elem_size(const epo_pool* p);
int epo_action_row_elems(const epo_pool* p);
/* teacher forcing (tests): read / overwrite one env's continuous state s[0..4], its
 * done flag and its step counters (current_step_ == elapsed_step_ for every env that has
 * one) without touching its RNG */
void epo_get_state(const epo_pool* p, int eid, double* s5, int* done, int* cur);
void epo_set_state(epo_pool* p, int eid, const double* s5, int done, int cur);
/* s[0..4] of every env at once: s5 is [num_envs][5] */
void epo_get_states(const epo_pool* p, double* s5);
/* toy_text teacher forcing of a whole pool (tests), RNG untouched: i8 is [num_envs][8]
 * integer state i[], done / cur one per env (elapsed_step_ = current_step_ = cur).  Blackjack's
 * hands: player32 / dealer32 [num_envs][32] cards with nplayer / ndealer counts; player32 NULL
 * leaves the hands (and the other three hand pointers unread) alone.  The getter fills the
 * same arrays. */
void epo_set_int_states(epo_pool* p, const int32_t* i8, const int32_t* player32,
                        const int32_t* nplayer, const int32_t* dealer32, const int32_t* ndealer,
                        const int32_t* done, const int32_t* cur);
void epo_get_int_states(const epo_pool* p, int32_t* i8, int32_t* player32, int32_t* nplayer,
                        int32_t* dealer32, int32_t* ndealer, int32_t* done, int32_t* cur);
/* HalfCheetah teacher forcing: s27 = qpos[9] qvel[9] qacc_warmstart[9] */
void epo_mjc_set(epo_pool* p, int eid, const double* s27, int done, int cur);
void epo_mjc_get(const epo_pool* p, int eid, double* s27);
/* raw engine draw from env `eid`'s std::mt19937 (for RNG known-answer tests) */
uint32_t epo_debug_draw(epo_pool* p, int eid);
void epo_debug_set_rng(epo_pool* p, int eid, const uint32_t* mt624, int idx);
void epo_debug_get_rng(const epo_pool* p, int eid, uint32_t* mt624, int* idx);
int epo_debug_uniform_int(epo_pool* p, int eid, int a, int b);
double epo_debug_uniform_real(epo_pool* p, int eid, double a, double b);
double epo_debug_normal(epo_pool* p, int eid, double mean, double stddev);

/* libm's sin and cos of n arguments, as the classic_control steps above take them: kind 0 =
 * double sin / cos, kind 1 = float sinf / cosf (x, s, c then point to floats).  s or c may be
 * NULL.  Returns 0, or -1 for an unknown kind. */
int epo_trig(int kind, const void* x, int n, void* s, void* c);

#ifdef __cplusplus
}
#endif
#endif /* EP_ORACLE_H_ */
