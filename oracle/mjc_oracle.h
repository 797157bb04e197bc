/* TEST INFRASTRUCTURE ONLY -- CPU restatement of the MuJoCo pipeline that the
 * reference's HalfCheetah env drives (envpool/mujoco/gym/mujoco_env.h:126-148).
 * See mjc_oracle.c for provenance and the PARITY UNPINNED notice. */
#ifndef MJC_ORACLE_H_
#define MJC_ORACLE_H_
#ifdef __cplusplus
extern "C" {
#endif

typedef struct mjc_model mjc_model;
typedef struct mjc_data mjc_data;
typedef double (*mjc_uniform_fn)(void* ctx, double a, double b);
typedef double (*mjc_normal_fn)(void* ctx, double mean, double stddev);

mjc_model* mjc_make_half_cheetah(void);
void mjc_free_model(mjc_model* m);
mjc_data* mjc_make_data(const mjc_model* m);
void mjc_free_data(mjc_data* d);
/* MujocoEnv::MujocoReset (mujoco_env.h:126-131) with HalfCheetah's
 * MujocoResetModel (half_cheetah.h:105-116): mj_resetData; qpos = init + U(-s,s);
 * qvel = init + N(0,s); mj_forward. */
void mjc_reset(const mjc_model* m, mjc_data* d, double noise_scale,
               mjc_uniform_fn uni, mjc_normal_fn nrm, void* ctx);
/* MujocoEnv::MujocoStep (mujoco_env.h:137-148), post_constraint=false (v4):
 * ctrl <- action; mj_step x frame_skip. */
void mjc_step(const mjc_model* m, mjc_data* d, const double* action, int frame_skip);
const double* mjc_qpos(const mjc_data* d);
const double* mjc_qvel(const mjc_data* d);
double* mjc_qpos_mut(mjc_data* d);
double* mjc_qvel_mut(mjc_data* d);
double* mjc_warm_mut(mjc_data* d); /* qacc_warmstart */
double* mjc_ctrl_mut(mjc_data* d); /* ctrl (mjc_step overwrites it with its action) */
/* mj_forward on the current qpos/qvel (used by tests to set a state) */
void mjc_forward(const mjc_model* m, mjc_data* d);
/* number of active constraint rows after the last forward/step (diagnostics) */
int mjc_nefc(const mjc_data* d);
/* dump compiled model constants as doubles into `out` (layout in mjc_oracle.c);
 * returns the count */
int mjc_model_constants(const mjc_model* m, double* out, int cap);

/* M(q) [81], bias(q, qvel) [9] (either may be NULL); returns the gravitational potential */
int mjc_debug_solve(const mjc_model* m, mjc_data* d, double* M_out, double* qfrc_smooth_out,
                    double* J_out, double* D_out, double* aref_out, int cap_rows,
                    double* qacc_out);
double mjc_debug_dynamics(const mjc_model* m, const double* qpos, const double* qvel,
                          double* M_out, double* bias_out);
/* Solver branch trace: from now on, (event, value) pairs of every branch the constraint solver
 * takes go to out[0 .. cap) (out = NULL: nowhere).  Returns the number of ints the previous
 * recording produced, which may exceed its cap.  Codes: mjc_oracle.c. */
int mjc_solver_trace(int* out, int cap);

#ifdef __cplusplus
}
#endif
#endif /* MJC_ORACLE_H_ */
