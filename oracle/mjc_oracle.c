/* TEST INFRASTRUCTURE ONLY -- CPU restatement of the physics behind the reference's
 * HalfCheetah env.
 *
 * PARITY UNPINNED.  The reference delegates all physics to MuJoCo 3.6.0
 * (envpool/workspace0.bzl:561-572; call sites envpool/mujoco/gym/mujoco_env.h:87,104,
 * 128-130,143), an un-vendored third-party C library that is absent from the reference tree
 * and from this image (no `mujoco` wheel, no network).  The reference's own tests for this
 * path (mujoco_gym_align_test.py, mujoco_gym_deterministic_test.py) hold no recorded
 * numbers.  This file therefore restates MuJoCo's *published* pipeline (documentation
 * chapters "Computation" and "Simulation", engine_forward / engine_core_constraint /
 * engine_solver as documented) for the one model on the hot path,
 * third_party/mujoco_gym_xml_patches/half_cheetah_envpool.xml, and is pinned only against
 * physical invariants (tests/test_mjc_oracle.py).  It is the parity target of the CUDA
 * HalfCheetah kernel, not a certified clone of MuJoCo; DESIGN.md lists the details that
 * must be re-verified once a MuJoCo 3.6.0 build is available (pyramidal R scaling,
 * diagApprox, line-search termination).
 *
 * The model is planar (every hinge axis is +y, the two root slides are x and z), so the
 * pipeline is written in the x-z plane: a body pose is (x, z, theta) with theta the
 * rotation about +y, R(theta) = [[c, s], [-s, c]] acting on (x, z).
 *
 * Pipeline per mj_step (mujoco_env.h:143), in MuJoCo's order:
 *   position  : kinematics, joint-space inertia M (+armature), collision (plane vs capsule
 *               end spheres), constraint rows (joint limits, pyramidal contacts)
 *   velocity  : passive forces (spring, damper), bias forces (Coriolis/centrifugal/gravity)
 *   actuation : ctrl clamped to ctrlrange, qfrc_actuator = gear * ctrl
 *   accel     : qacc_smooth = M^-1 (passive - bias + actuator)
 *   constraint: Newton solver on the convex primal problem, warm-started
 *   integrate : semi-implicit Euler with implicit joint damping
 */
#include "mjc_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define NV 9
#define NB 7  /* moving bodies: torso bthigh bshin bfoot fthigh fshin ffoot */
#define NG 8  /* capsule geoms */
#define NU 6
#define MAXCON 16
#define MAXROW (6 + 4 * MAXCON)
#define MJ_MINVAL 1e-15
#define MJ_MINIMP 0.0001
#define MJ_MAXIMP 0.9999

struct mjc_model {
  int parent[NB];        /* -1 = world */
  double bpos[NB][2];    /* body frame origin in the parent frame (x, z) */
  double mass[NB], com[NB][2], iyy[NB];
  int body_dof[NB];      /* dof of the body's own hinge */
  double armature[NV], damping[NV], stiffness[NV], range[NV][2];
  int limited[NV];
  double gear[NU];
  int gbody[NG];
  double gpos[NG][2], gaxis[NG][2], ghalf[NG], grad;
  double timestep, gravity, mu;
  double solref[2], solimp[3], solref_limit[2], solimp_limit[3];
  double dof_invweight0[NV], body_invweight0[NB][2], meaninertia;
  double torso_z0;
  double tolerance;
  int max_iter, ls_iter;
};

struct mjc_data {
  double qpos[NV], qvel[NV], ctrl[NU], qacc_warmstart[NV], qacc[NV];
  int nefc, ncon, niter;
};

/* ------------------------------------------------------------- small dense algebra --- */
static int chol9(const double* A, double* L) { /* A = L L^T, row-major NVxNV */
  memcpy(L, A, sizeof(double) * NV * NV);
  for (int j = 0; j < NV; ++j) {
    double d = L[j * NV + j];
    for (int k = 0; k < j; ++k) d -= L[j * NV + k] * L[j * NV + k];
    if (d <= 0) return -1;
    d = sqrt(d);
    L[j * NV + j] = d;
    for (int i = j + 1; i < NV; ++i) {
      double s = L[i * NV + j];
      for (int k = 0; k < j; ++k) s -= L[i * NV + k] * L[j * NV + k];
      L[i * NV + j] = s / d;
    }
  }
  return 0;
}
static void chol_solve9(const double* L, const double* b, double* x) {
  double y[NV];
  for (int i = 0; i < NV; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= L[i * NV + k] * y[k];
    y[i] = s / L[i * NV + i];
  }
  for (int i = NV - 1; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < NV; ++k) s -= L[k * NV + i] * x[k];
    x[i] = s / L[i * NV + i];
  }
}
static void matvec9(const double* A, const double* x, double* y) {
  for (int i = 0; i < NV; ++i) {
    double s = 0;
    for (int k = 0; k < NV; ++k) s += A[i * NV + k] * x[k];
    y[i] = s;
  }
}

/* ------------------------------------------------------------------ model compile --- */
static void capsule_inertia(double r, double h, double density, double* mass,
                            double* itrans) {
  /* MuJoCo compiler, capsule = cylinder (length 2h) + two hemispheres; inertia about the
   * centre for an axis perpendicular to the capsule axis */
  double height = 2 * h;
  double mc = density * M_PI * r * r * height;
  double ms = density * 4.0 / 3.0 * M_PI * r * r * r;
  *mass = mc + ms;
  *itrans = mc * (3 * r * r + height * height) / 12.0 +
            ms * (0.4 * r * r + 0.375 * r * height + 0.25 * height * height);
}

static void set_geom_axisangle(mjc_model* m, int g, int body, double px, double pz,
                               double angle, double half) {
  m->gbody[g] = body;
  m->gpos[g][0] = px;
  m->gpos[g][1] = pz;
  /* geom z-axis after rotating by `angle` about +y: (sin a, cos a) in (x, z) */
  m->gaxis[g][0] = sin(angle);
  m->gaxis[g][1] = cos(angle);
  m->ghalf[g] = half;
}

/* forward declarations */
static void kinematics(const mjc_model* m, const double* q, double org[NB][2],
                       double th[NB], double com[NB][2]);
static void mass_matrix(const mjc_model* m, double org[NB][2], double com[NB][2],
                        double* M);
static void point_jac(const mjc_model* m, int body, const double p[2], double org[NB][2],
                      double* Jx, double* Jz);

mjc_model* mjc_make_half_cheetah(void) {
  mjc_model* m = (mjc_model*)calloc(1, sizeof(mjc_model));
  /* kinematic tree, half_cheetah_envpool.xml:71-102 */
  const int parent[NB] = {-1, 0, 1, 2, 0, 4, 5};
  const double bpos[NB][2] = {{0, 0.7},     {-0.5, 0},   {0.16, -0.25}, {-0.28, -0.14},
                              {0.5, 0},     {-0.14, -0.24}, {0.13, -0.18}};
  for (int b = 0; b < NB; ++b) {
    m->parent[b] = parent[b];
    m->bpos[b][0] = bpos[b][0];
    m->bpos[b][1] = bpos[b][1];
    m->body_dof[b] = b + 2; /* torso hinge rooty = dof 2, limb hinges 3..8 */
  }
  m->torso_z0 = 0.7;
  /* joints: rootx rootz rooty have armature=damping=stiffness=0, unlimited (xml:72-74);
   * limb hinges: default armature .1, per-joint damping/stiffness/range (xml:54,79-97) */
  const double damp[6] = {6, 4.5, 3, 4.5, 3, 1.5};
  const double stiff[6] = {240, 180, 120, 180, 120, 60};
  const double range[6][2] = {{-.52, 1.05}, {-.785, .785}, {-.4, .785},
                              {-1, .7},     {-1.2, .87},   {-.5, .5}};
  const double gear[NU] = {120, 90, 60, 120, 60, 30};
  for (int j = 0; j < 6; ++j) {
    m->armature[3 + j] = 0.1;
    m->damping[3 + j] = damp[j];
    m->stiffness[3 + j] = stiff[j];
    m->range[3 + j][0] = range[j][0];
    m->range[3 + j][1] = range[j][1];
    m->limited[3 + j] = 1;
    m->gear[j] = gear[j];
  }
  /* geoms (xml:75-76,80,83,86,92,95,98); all capsules, radius 0.046 */
  m->grad = 0.046;
  m->gbody[0] = 0; /* torso: fromto -.5 0 0 .5 0 0 */
  m->gpos[0][0] = 0; m->gpos[0][1] = 0; m->gaxis[0][0] = 1; m->gaxis[0][1] = 0;
  m->ghalf[0] = 0.5;
  set_geom_axisangle(m, 1, 0, 0.6, 0.1, 0.87, 0.15);      /* head */
  set_geom_axisangle(m, 2, 1, 0.1, -0.13, -3.8, 0.145);   /* bthigh */
  set_geom_axisangle(m, 3, 2, -0.14, -0.07, -2.03, 0.15); /* bshin */
  set_geom_axisangle(m, 4, 3, 0.03, -0.097, -0.27, 0.094);/* bfoot */
  set_geom_axisangle(m, 5, 4, -0.07, -0.12, 0.52, 0.133); /* fthigh */
  set_geom_axisangle(m, 6, 5, 0.065, -0.09, -0.6, 0.106); /* fshin */
  set_geom_axisangle(m, 7, 6, 0.045, -0.07, -0.6, 0.07);  /* ffoot */
  /* inertiafromgeom: density 1000, then settotalmass=14 (xml:52) */
  double gm[NG], gi[NG], total = 0;
  for (int g = 0; g < NG; ++g) {
    capsule_inertia(m->grad, m->ghalf[g], 1000.0, &gm[g], &gi[g]);
    total += gm[g];
  }
  for (int b = 0; b < NB; ++b) {
    double mb = 0, cx = 0, cz = 0;
    for (int g = 0; g < NG; ++g)
      if (m->gbody[g] == b) {
        mb += gm[g];
        cx += gm[g] * m->gpos[g][0];
        cz += gm[g] * m->gpos[g][1];
      }
    cx /= mb;
    cz /= mb;
    double iyy = 0;
    for (int g = 0; g < NG; ++g)
      if (m->gbody[g] == b) {
        double dx = m->gpos[g][0] - cx, dz = m->gpos[g][1] - cz;
        iyy += gi[g] + gm[g] * (dx * dx + dz * dz);
      }
    double scale = 14.0 / total;
    m->mass[b] = mb * scale;
    m->com[b][0] = cx;
    m->com[b][1] = cz;
    m->iyy[b] = iyy * scale;
  }
  /* option / defaults (xml:54-59): timestep .01, gravity -9.81, friction .4 (max of the two
   * geoms, both .4), contact solref .02 1 solimp 0 .8 .01, limit solref .02 1 solimp 0 .8 .03;
   * MuJoCo defaults: Newton, 100 iterations, tolerance 1e-8, 50 line-search iterations */
  m->timestep = 0.01;
  m->gravity = -9.81;
  m->mu = 0.4;
  m->solref[0] = 0.02; m->solref[1] = 1;
  m->solimp[0] = 0.0; m->solimp[1] = 0.8; m->solimp[2] = 0.01;
  m->solref_limit[0] = 0.02; m->solref_limit[1] = 1;
  m->solimp_limit[0] = 0.0; m->solimp_limit[1] = 0.8; m->solimp_limit[2] = 0.03;
  m->tolerance = 1e-8;
  m->max_iter = 100;
  m->ls_iter = 50;
  /* mj_setConst at qpos0: inverse weights and mean inertia */
  double q0[NV] = {0}, org[NB][2], th[NB], com[NB][2], M[NV * NV], L[NV * NV];
  kinematics(m, q0, org, th, com);
  mass_matrix(m, org, com, M);
  chol9(M, L);
  double Minv[NV * NV];
  for (int j = 0; j < NV; ++j) {
    double e[NV] = {0}, x[NV];
    e[j] = 1;
    chol_solve9(L, e, x);
    for (int i = 0; i < NV; ++i) Minv[i * NV + j] = x[i];
  }
  double tr = 0;
  for (int i = 0; i < NV; ++i) {
    m->dof_invweight0[i] = Minv[i * NV + i];
    tr += M[i * NV + i];
  }
  m->meaninertia = tr / NV;
  for (int b = 0; b < NB; ++b) {
    /* translational: trace(Jp Minv Jp^T)/3 at the body CoM (the y row is identically 0 in
     * this planar model); rotational: (Jr Minv Jr^T)_yy / 3 */
    double Jx[NV], Jz[NV], Jr[NV] = {0}, t[NV];
    point_jac(m, b, com[b], org, Jx, Jz);
    for (int a = b; a >= 0; a = m->parent[a]) Jr[m->body_dof[a]] = 1;
    double axx = 0, azz = 0, arr = 0;
    matvec9(Minv, Jx, t);
    for (int i = 0; i < NV; ++i) axx += Jx[i] * t[i];
    matvec9(Minv, Jz, t);
    for (int i = 0; i < NV; ++i) azz += Jz[i] * t[i];
    matvec9(Minv, Jr, t);
    for (int i = 0; i < NV; ++i) arr += Jr[i] * t[i];
    m->body_invweight0[b][0] = (axx + azz) / 3.0;
    m->body_invweight0[b][1] = arr / 3.0;
  }
  return m;
}

void mjc_free_model(mjc_model* m) { free(m); }
mjc_data* mjc_make_data(const mjc_model* m) {
  (void)m;
  return (mjc_data*)calloc(1, sizeof(mjc_data));
}
void mjc_free_data(mjc_data* d) { free(d); }
const double* mjc_qpos(const mjc_data* d) { return d->qpos; }
const double* mjc_qvel(const mjc_data* d) { return d->qvel; }
double* mjc_qpos_mut(mjc_data* d) { return d->qpos; }
double* mjc_qvel_mut(mjc_data* d) { return d->qvel; }
double* mjc_warm_mut(mjc_data* d) { return d->qacc_warmstart; }
double* mjc_ctrl_mut(mjc_data* d) { return d->ctrl; }
int mjc_nefc(const mjc_data* d) { return d->nefc; }

int mjc_model_constants(const mjc_model* m, double* out, int cap) {
  int n = 0;
#define PUT(v) do { if (n < cap) out[n] = (v); ++n; } while (0)
  for (int b = 0; b < NB; ++b) { PUT(m->mass[b]); PUT(m->com[b][0]); PUT(m->com[b][1]); PUT(m->iyy[b]); }
  for (int i = 0; i < NV; ++i) PUT(m->dof_invweight0[i]);
  for (int b = 0; b < NB; ++b) { PUT(m->body_invweight0[b][0]); PUT(m->body_invweight0[b][1]); }
  PUT(m->meaninertia);
#undef PUT
  return n;
}

/* ---------------------------------------------------------------------- kinematics --- */
/* world pose of every body frame and CoM.  R(theta) (x,z) = (c x + s z, -s x + c z). */
static void kinematics(const mjc_model* m, const double* q, double org[NB][2],
                       double th[NB], double com[NB][2]) {
  for (int b = 0; b < NB; ++b) {
    if (m->parent[b] < 0) {
      org[b][0] = m->bpos[b][0] + q[0];
      org[b][1] = m->bpos[b][1] + q[1];
      th[b] = q[2];
    } else {
      int p = m->parent[b];
      double c = cos(th[p]), s = sin(th[p]);
      org[b][0] = org[p][0] + c * m->bpos[b][0] + s * m->bpos[b][1];
      org[b][1] = org[p][1] - s * m->bpos[b][0] + c * m->bpos[b][1];
      th[b] = th[p] + q[m->body_dof[b]];
    }
    double c = cos(th[b]), s = sin(th[b]);
    com[b][0] = org[b][0] + c * m->com[b][0] + s * m->com[b][1];
    com[b][1] = org[b][1] - s * m->com[b][0] + c * m->com[b][1];
  }
}

/* Jacobian of the world velocity (x, z) of point p fixed to `body`.  A hinge about +y at
 * origin o moves p with omega * (r_z, -r_x), r = p - o. */
static void point_jac(const mjc_model* m, int body, const double p[2], double org[NB][2],
                      double* Jx, double* Jz) {
  for (int i = 0; i < NV; ++i) Jx[i] = Jz[i] = 0;
  Jx[0] = 1;
  Jz[1] = 1;
  for (int a = body; a >= 0; a = m->parent[a]) {
    int d = m->body_dof[a];
    Jx[d] = p[1] - org[a][1];
    Jz[d] = -(p[0] - org[a][0]);
  }
}

/* joint-space inertia: M = sum_b m_b Jc^T Jc + I_b Jr^T Jr + diag(armature)  (what the
 * composite-rigid-body pass of mj_crb produces) */
static void mass_matrix(const mjc_model* m, double org[NB][2], double com[NB][2],
                        double* M) {
  memset(M, 0, sizeof(double) * NV * NV);
  for (int b = 0; b < NB; ++b) {
    double Jx[NV], Jz[NV], Jr[NV] = {0};
    point_jac(m, b, com[b], org, Jx, Jz);
    for (int a = b; a >= 0; a = m->parent[a]) Jr[m->body_dof[a]] = 1;
    for (int i = 0; i < NV; ++i)
      for (int j = 0; j < NV; ++j)
        M[i * NV + j] += m->mass[b] * (Jx[i] * Jx[j] + Jz[i] * Jz[j]) + m->iyy[b] * Jr[i] * Jr[j];
  }
  for (int i = 0; i < NV; ++i) M[i * NV + i] += m->armature[i];
}

/* bias force (mj_rne with zero acceleration): Coriolis/centrifugal + gravity.
 * With qacc = 0 the CoM acceleration of body b is the sum of centripetal terms
 * -omega_a^2 * r along its ancestor chain; angular acceleration is zero in the plane. */
static void bias_force(const mjc_model* m, const double* qv, double org[NB][2],
                       double com[NB][2], double* bias) {
  double omega[NB], aorg[NB][2];
  for (int b = 0; b < NB; ++b) {
    int p = m->parent[b];
    if (p < 0) {
      omega[b] = qv[2];
      aorg[b][0] = aorg[b][1] = 0;
    } else {
      omega[b] = omega[p] + qv[m->body_dof[b]];
      double rx = org[b][0] - org[p][0], rz = org[b][1] - org[p][1];
      aorg[b][0] = aorg[p][0] - omega[p] * omega[p] * rx;
      aorg[b][1] = aorg[p][1] - omega[p] * omega[p] * rz;
    }
  }
  for (int i = 0; i < NV; ++i) bias[i] = 0;
  for (int b = 0; b < NB; ++b) {
    double rx = com[b][0] - org[b][0], rz = com[b][1] - org[b][1];
    double ax = aorg[b][0] - omega[b] * omega[b] * rx;
    double az = aorg[b][1] - omega[b] * omega[b] * rz - m->gravity; /* a - g */
    double Jx[NV], Jz[NV];
    point_jac(m, b, com[b], org, Jx, Jz);
    for (int i = 0; i < NV; ++i) bias[i] += m->mass[b] * (Jx[i] * ax + Jz[i] * az);
  }
}

/* ---------------------------------------------------------------------- constraints --- */
typedef struct {
  int n;
  double J[MAXROW][NV];
  double pos[MAXROW], D[MAXROW], aref[MAXROW];
} efc_t;

/* getimpedance + K,B (mj_makeImpedance): returns imp, K, B */
static void impedance(const double* solref, const double* solimp, double pos, double* imp,
                      double* K, double* B) {
  double dmin = fmin(MJ_MAXIMP, fmax(MJ_MINIMP, solimp[0]));
  double dmax = fmin(MJ_MAXIMP, fmax(MJ_MINIMP, solimp[1]));
  double width = solimp[2], mid = 0.5, power = 2;
  double x = fabs(pos) / width, y;
  if (x >= 1) {
    *imp = dmax;
  } else if (x <= 0) {
    *imp = dmin;
  } else {
    if (x <= mid) {
      y = pow(x, power) / pow(mid, power - 1);
    } else {
      y = 1 - pow(1 - x, power) / pow(1 - mid, power - 1);
    }
    *imp = dmin + y * (dmax - dmin);
  }
  *K = 1 / fmax(MJ_MINVAL, dmax * dmax * solref[0] * solref[0] * solref[1] * solref[1]);
  *B = 2 / fmax(MJ_MINVAL, dmax * solref[0]);
}

static void add_row(efc_t* e, const double* J, double pos, double diagApprox,
                    const double* solref, const double* solimp, const double* qv,
                    double Rscale) {
  int r = e->n++;
  double imp, K, B, vel = 0;
  memcpy(e->J[r], J, sizeof(double) * NV);
  for (int i = 0; i < NV; ++i) vel += J[i] * qv[i];
  impedance(solref, solimp, pos, &imp, &K, &B);
  double R = fmax(MJ_MINVAL, (1 - imp) * diagApprox / imp) * Rscale;
  e->pos[r] = pos;
  e->D[r] = 1 / R;
  e->aref[r] = -B * vel - K * imp * pos;
}

static void make_constraints(const mjc_model* m, const double* q, const double* qv,
                             double org[NB][2], double th[NB], efc_t* e, int* ncon) {
  e->n = 0;
  *ncon = 0;
  /* joint limits (mj_instantiateLimit): side -1 then +1, dist = side*(range - q) */
  for (int i = 0; i < NV; ++i) {
    if (!m->limited[i]) continue;
    for (int side = -1; side <= 1; side += 2) {
      double dist = side * (m->range[i][(side + 1) / 2] - q[i]);
      if (dist < 0) {
        double J[NV] = {0};
        J[i] = -side;
        add_row(e, J, dist, m->dof_invweight0[i], m->solref_limit, m->solimp_limit, qv, 1.0);
      }
    }
  }
  /* contacts: floor plane (z = 0, normal +z) vs the two end spheres of every capsule
   * (mjc_PlaneCapsule -> _PlaneSphere), margin 0; condim 3, pyramidal cone:
   * rows n + mu t1, n - mu t1, n + mu t2, n - mu t2 with t1 = +-x, t2 = +-y.  The model
   * never moves along y, so the two t2 rows equal the normal row. */
  for (int g = 0; g < NG; ++g) {
    int b = m->gbody[g];
    double c = cos(th[b]), s = sin(th[b]);
    double cx = org[b][0] + c * m->gpos[g][0] + s * m->gpos[g][1];
    double cz = org[b][1] - s * m->gpos[g][0] + c * m->gpos[g][1];
    double ax = c * m->gaxis[g][0] + s * m->gaxis[g][1];
    double az = -s * m->gaxis[g][0] + c * m->gaxis[g][1];
    for (int end = 1; end >= -1; end -= 2) {
      double px = cx + end * m->ghalf[g] * ax, pz = cz + end * m->ghalf[g] * az;
      double dist = pz - m->grad;
      if (pz > m->grad) continue; /* cdist > margin + radius */
      if (*ncon >= MAXCON) continue;
      ++*ncon;
      /* contact point: sphere centre - n * (radius + dist/2) */
      double p[2] = {px, pz - (m->grad + dist / 2)};
      double Jx[NV], Jz[NV], row[NV];
      point_jac(m, b, p, org, Jx, Jz);
      /* mj_diagApprox, pyramidal: tran + mu^2 * tran (translational weights of both
       * bodies; the world body weighs 0).  R of every edge = 2 mu^2 R(first edge). */
      double tran = m->body_invweight0[b][0];
      double dA = tran + m->mu * m->mu * tran;
      double Rscale = 2 * m->mu * m->mu;
      for (int i = 0; i < NV; ++i) row[i] = Jz[i] + m->mu * Jx[i];
      add_row(e, row, dist, dA, m->solref, m->solimp, qv, Rscale);
      for (int i = 0; i < NV; ++i) row[i] = Jz[i] - m->mu * Jx[i];
      add_row(e, row, dist, dA, m->solref, m->solimp, qv, Rscale);
      add_row(e, Jz, dist, dA, m->solref, m->solimp, qv, Rscale);
      add_row(e, Jz, dist, dA, m->solref, m->solimp, qv, Rscale);
    }
  }
}

/* ------------------------------------------------------------------------- solver --- */
static long g_ls_hist[64]; /* diagnostics: histogram of line-search evaluations per Newton step */
void mjc_debug_ls_hist(long* out) { for (int i = 0; i < 64; ++i) { out[i] = g_ls_hist[i]; g_ls_hist[i] = 0; } }

/* Solver branch trace: (event, value) pairs with the event and value codes of the pair kernel's
 * host test build (envpool_b200/csrc/mujoco_pair.cuh, HCP_STATS), plus TR_CONTACTS.  Recorded
 * only while mjc_solver_trace has been given a buffer. */
enum { TR_ROWS = 1, TR_WARM, TR_LS, TR_UPD, TR_LS_END, TR_EXIT, TR_CONTACTS };
enum { TR_RUN = 0 };
enum { TR_NEWTON = 0, TR_EXPAND, TR_BISECT };
enum { TR_CONV = 0, TR_STALL, TR_CAP };
enum { TR_GRAD0 = 0, TR_COST, TR_GRAD, TR_MAXITER, TR_ALPHA0 };
static int* g_trace;
static int g_trace_cap, g_trace_len;
static void trace(int ev, int val) {
  if (!g_trace) return;
  if (g_trace_len + 2 <= g_trace_cap) {
    g_trace[g_trace_len] = ev;
    g_trace[g_trace_len + 1] = val;
  }
  g_trace_len += 2;
}
int mjc_solver_trace(int* out, int cap) {
  const int n = g_trace_len;
  g_trace = out;
  g_trace_cap = out ? cap : 0;
  g_trace_len = 0;
  return n;
}
/* cost(a) = 1/2 (a - a_s)^T M (a - a_s) + sum_i 1/2 D_i min(0, J_i a - aref_i)^2 */
static double constraint_cost(const efc_t* e, const double* jar) {
  double c = 0;
  for (int r = 0; r < e->n; ++r)
    if (jar[r] < 0) c += 0.5 * e->D[r] * jar[r] * jar[r];
  return c;
}

static void solve_newton(const mjc_model* m, const efc_t* e, const double* M,
                         const double* qfrc_smooth, const double* qacc_smooth,
                         const double* warm, double* qacc, double* qfrc_constraint,
                         int* niter) {
  const int n = e->n;
  double jar[MAXROW], Ma[NV], grad[NV], search[NV], Mv[NV], Jv[MAXROW];
  *niter = 0;
  if (n == 0) {
    memcpy(qacc, qacc_smooth, sizeof(double) * NV);
    memset(qfrc_constraint, 0, sizeof(double) * NV);
    return;
  }
  /* warmstart (engine_forward.c): keep qacc_warmstart only if its total cost beats the
   * cost at qacc_smooth */
  {
    double cw, cs;
    for (int r = 0; r < n; ++r) {
      double s = -e->aref[r];
      for (int i = 0; i < NV; ++i) s += e->J[r][i] * warm[i];
      jar[r] = s;
    }
    cw = constraint_cost(e, jar);
    matvec9(M, warm, Ma);
    for (int i = 0; i < NV; ++i) cw += 0.5 * (Ma[i] - qfrc_smooth[i]) * (warm[i] - qacc_smooth[i]);
    for (int r = 0; r < n; ++r) {
      double s = -e->aref[r];
      for (int i = 0; i < NV; ++i) s += e->J[r][i] * qacc_smooth[i];
      jar[r] = s;
    }
    cs = constraint_cost(e, jar);
    memcpy(qacc, cw > cs ? qacc_smooth : warm, sizeof(double) * NV);
    trace(TR_WARM, (cw > cs ? 1 : 0) + (cw == cs ? 2 : 0));
  }
  const double scale = 1.0 / (m->meaninertia * NV);
  double cost = 0;
  for (int iter = 0; iter <= m->max_iter; ++iter) {
    /* constraint update at the current point */
    matvec9(M, qacc, Ma);
    double H[NV * NV], L[NV * NV];
    memcpy(H, M, sizeof(H));
    for (int i = 0; i < NV; ++i) qfrc_constraint[i] = 0;
    double newcost = 0;
    for (int r = 0; r < n; ++r) {
      double s = -e->aref[r];
      for (int i = 0; i < NV; ++i) s += e->J[r][i] * qacc[i];
      jar[r] = s;
      if (s < 0) {
        double f = -e->D[r] * s;
        newcost += 0.5 * e->D[r] * s * s;
        for (int i = 0; i < NV; ++i) {
          qfrc_constraint[i] += e->J[r][i] * f;
          for (int j = 0; j < NV; ++j) H[i * NV + j] += e->D[r] * e->J[r][i] * e->J[r][j];
        }
      }
    }
    for (int i = 0; i < NV; ++i)
      newcost += 0.5 * (Ma[i] - qfrc_smooth[i]) * (qacc[i] - qacc_smooth[i]);
    double gnorm = 0;
    for (int i = 0; i < NV; ++i) {
      grad[i] = Ma[i] - qfrc_smooth[i] - qfrc_constraint[i];
      gnorm += grad[i] * grad[i];
    }
    gnorm = sqrt(gnorm);
    if (iter > 0) {
      double improvement = scale * (cost - newcost);
      if (improvement < m->tolerance || scale * gnorm < m->tolerance) {
        trace(TR_EXIT, improvement < m->tolerance ? TR_COST : TR_GRAD);
        cost = newcost;
        break;
      }
    } else if (scale * gnorm < m->tolerance) {
      trace(TR_EXIT, TR_GRAD0);
      break;
    }
    cost = newcost;
    if (iter == m->max_iter) {
      trace(TR_EXIT, TR_MAXITER);
      break;
    }
    ++*niter;
    /* Newton direction */
    chol9(H, L);
    chol_solve9(L, grad, search);
    for (int i = 0; i < NV; ++i) search[i] = -search[i];
    /* exact line search on the convex piecewise-quadratic phi(alpha): safeguarded Newton
     * on phi'(alpha) */
    matvec9(M, search, Mv);
    for (int r = 0; r < n; ++r) {
      double s = 0;
      for (int i = 0; i < NV; ++i) s += e->J[r][i] * search[i];
      Jv[r] = s;
    }
    double q1 = 0, q2 = 0; /* Gauss part: phi_g'(alpha) = q1 + alpha*q2 */
    for (int i = 0; i < NV; ++i) {
      q1 += search[i] * (Ma[i] - qfrc_smooth[i]);
      q2 += search[i] * Mv[i];
    }
    /* stop when |phi'(alpha)| < tolerance * ls_tolerance * |search| / scale (MuJoCo's
     * scaled gradient tolerance for the 1-D problem; ls_tolerance = 0.01) */
    double snorm = 0;
    for (int i = 0; i < NV; ++i) snorm += search[i] * search[i];
    const double gtol = m->tolerance * 0.01 * sqrt(snorm) / scale;
    double lo = 0, hi = INFINITY, alpha = 0;
    int ls_evals = 0, ls_end = TR_CAP;
    trace(TR_LS, TR_RUN);
    for (int k = 0; k < m->ls_iter; ++k) {
      ++ls_evals;
      double d1 = q1 + alpha * q2, d2 = q2;
      for (int r = 0; r < n; ++r) {
        double x = jar[r] + alpha * Jv[r];
        if (x < 0) {
          d1 += e->D[r] * x * Jv[r];
          d2 += e->D[r] * Jv[r] * Jv[r];
        }
      }
      if (fabs(d1) < gtol) {
        ls_end = TR_CONV;
        break;
      }
      if (d1 < 0) lo = alpha; else hi = alpha;
      double next = alpha - d1 / d2;
      const int upd = (next > lo && next < hi) ? TR_NEWTON : (isinf(hi) ? TR_EXPAND : TR_BISECT);
      if (!(next > lo && next < hi)) next = isinf(hi) ? 2 * alpha + 1 : 0.5 * (lo + hi);
      if (next == alpha) {
        ls_end = TR_STALL;
        break;
      }
      trace(TR_UPD, upd);
      alpha = next;
    }
    trace(TR_LS_END, ls_end);
    g_ls_hist[ls_evals < 63 ? ls_evals : 63]++;
    if (alpha == 0) {
      trace(TR_EXIT, TR_ALPHA0);
      break;
    }
    for (int i = 0; i < NV; ++i) qacc[i] += alpha * search[i];
  }
}

/* ---------------------------------------------------------------- forward and step --- */
static void forward(const mjc_model* m, mjc_data* d, double* M, double* qfrc_smooth,
                    double* qfrc_constraint) {
  double org[NB][2], th[NB], com[NB][2], bias[NV], L[NV * NV], qacc_smooth[NV];
  static efc_t e; /* single-threaded test infrastructure */
  kinematics(m, d->qpos, org, th, com);
  mass_matrix(m, org, com, M);
  make_constraints(m, d->qpos, d->qvel, org, th, &e, &d->ncon);
  bias_force(m, d->qvel, org, com, bias);
  for (int i = 0; i < NV; ++i) {
    /* passive: spring toward qpos0 = 0 and damper (mj_passive) */
    double passive = -m->stiffness[i] * d->qpos[i] - m->damping[i] * d->qvel[i];
    double act = 0;
    if (i >= 3) {
      double c = d->ctrl[i - 3];
      c = c < -1 ? -1 : (c > 1 ? 1 : c); /* ctrllimited, ctrlrange -1 1 */
      act = m->gear[i - 3] * c;
    }
    qfrc_smooth[i] = passive - bias[i] + act;
  }
  chol9(M, L);
  chol_solve9(L, qfrc_smooth, qacc_smooth);
  d->nefc = e.n;
  trace(TR_ROWS, e.n);
  trace(TR_CONTACTS, d->ncon);
  solve_newton(m, &e, M, qfrc_smooth, qacc_smooth, d->qacc_warmstart, d->qacc,
               qfrc_constraint, &d->niter);
}

/* Diagnostics for tests/test_mjc_oracle.py: joint-space inertia M(q) (row-major NVxNV), bias
 * force c(q, qvel) (Coriolis/centrifugal + gravity) and the gravitational potential
 * V(q) = sum_b m_b |g| z_com,b -- enough to check the bias against Lagrange's equations,
 * c_i = sum_jk (dM_ij/dq_k - 1/2 dM_jk/dq_i) v_j v_k + dV/dq_i, by finite differences. */
double mjc_debug_dynamics(const mjc_model* m, const double* qpos, const double* qvel,
                          double* M_out, double* bias_out) {
  double org[NB][2], th[NB], com[NB][2], V = 0;
  kinematics(m, qpos, org, th, com);
  if (M_out) mass_matrix(m, org, com, M_out);
  if (bias_out) bias_force(m, qvel, org, com, bias_out);
  for (int b = 0; b < NB; ++b) V -= m->mass[b] * m->gravity * com[b][1]; /* gravity < 0 */
  return V;
}

/* Diagnostics for tests/test_mjc_oracle.py: the constraint problem of the current state as the
 * solver sees it -- M (row-major NVxNV), qfrc_smooth, the rows (J row-major [n][NV], D, aref)
 * -- and the solver's answer qacc, so that an independent optimiser can be run on the same
 * convex cost  1/2 (a - a_s)' M (a - a_s) + sum_i 1/2 D_i min(0, J_i a - aref_i)^2.  Returns the
 * number of rows (at most cap_rows are written). */
int mjc_debug_solve(const mjc_model* m, mjc_data* d, double* M_out, double* qfrc_smooth_out,
                    double* J_out, double* D_out, double* aref_out, int cap_rows,
                    double* qacc_out) {
  double org[NB][2], th[NB], com[NB][2];
  double M[NV * NV], fs[NV], fc[NV];
  static efc_t e;
  int ncon = 0;
  forward(m, d, M, fs, fc);
  kinematics(m, d->qpos, org, th, com);
  make_constraints(m, d->qpos, d->qvel, org, th, &e, &ncon);
  memcpy(M_out, M, sizeof(M));
  memcpy(qfrc_smooth_out, fs, sizeof(fs));
  memcpy(qacc_out, d->qacc, sizeof(double) * NV);
  for (int r = 0; r < e.n && r < cap_rows; ++r) {
    memcpy(J_out + r * NV, e.J[r], sizeof(double) * NV);
    D_out[r] = e.D[r];
    aref_out[r] = e.aref[r];
  }
  return e.n;
}

void mjc_forward(const mjc_model* m, mjc_data* d) {
  double M[NV * NV], fs[NV], fc[NV];
  forward(m, d, M, fs, fc);
}

static void step1(const mjc_model* m, mjc_data* d) {
  double M[NV * NV], fs[NV], fc[NV], rhs[NV], qacc[NV], L[NV * NV];
  forward(m, d, M, fs, fc);
  /* mj_Euler with implicit joint damping: (M + h diag(damping)) a = qfrc_smooth +
   * qfrc_constraint; qvel += h a; qpos += h qvel */
  for (int i = 0; i < NV; ++i) {
    M[i * NV + i] += m->timestep * m->damping[i];
    rhs[i] = fs[i] + fc[i];
  }
  chol9(M, L);
  chol_solve9(L, rhs, qacc);
  for (int i = 0; i < NV; ++i) d->qvel[i] += m->timestep * qacc[i];
  for (int i = 0; i < NV; ++i) d->qpos[i] += m->timestep * d->qvel[i];
  memcpy(d->qacc_warmstart, d->qacc, sizeof(double) * NV); /* mj_advance */
}

void mjc_step(const mjc_model* m, mjc_data* d, const double* action, int frame_skip) {
  for (int i = 0; i < NU; ++i) d->ctrl[i] = action[i];
  for (int k = 0; k < frame_skip; ++k) step1(m, d);
}

void mjc_reset(const mjc_model* m, mjc_data* d, double noise_scale, mjc_uniform_fn uni,
               mjc_normal_fn nrm, void* ctx) {
  /* mj_resetData: qpos = qpos0 (all zero for this model: slides/hinges, no ref), qvel = 0,
   * ctrl = 0, qacc_warmstart = 0 */
  memset(d, 0, sizeof(*d));
  for (int i = 0; i < NV; ++i) d->qpos[i] = 0.0 + uni(ctx, -noise_scale, noise_scale);
  for (int i = 0; i < NV; ++i) d->qvel[i] = 0.0 + nrm(ctx, 0.0, noise_scale);
  /* mj_forward has no lasting effect on (qpos, qvel, qacc_warmstart); run it anyway so the
   * diagnostics (nefc) describe the reset state */
  mjc_forward(m, d);
}
