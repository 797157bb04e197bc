// HalfCheetah (mujoco/gym) family.  The reference's per-env Step() is
//   ctrl <- action; mj_step x frame_skip        (envpool/mujoco/gym/mujoco_env.h:137-148)
//   reward / obs / infos from qpos, qvel        (envpool/mujoco/gym/half_cheetah.h:136-185)
// with all physics inside MuJoCo 3.6.0 (third-party, not vendored).  This file is a
// from-scratch CUDA formulation of MuJoCo's documented pipeline for the one model on the
// path, third_party/mujoco_gym_xml_patches/half_cheetah_envpool.xml: planar kinematic tree
// (nq = nv = 9, 7 moving bodies, 8 capsules, floor plane), joint-space inertia, bias forces,
// joint-limit + pyramidal-contact constraint rows, Newton solver with exact line search on
// the convex primal problem, semi-implicit Euler with implicit joint damping.
//
// Three kernels, selected by ENVPOOL_B200_HC_KERNEL at pool creation:
//   pair   (default)  two lanes per env, mujoco_pair.cuh -- hc_pair_kernel below
//   thread            one thread per env, mujoco_thread.cuh -- hc_thread_kernel
//   warp              one warp per env, this file -- hc_kernel: lanes are bodies (kinematics),
//                     matrix entries (inertia, Hessian), candidate contacts / limits (collision),
//                     constraint rows (solver); 9x9 systems, row table and per-step vectors in
//                     shared memory (9 KB per warp), warp-shuffle reductions.  What north_star
//                     suggested; 9x slower than thread-per-env because nv = 9 cannot feed 32 lanes.
// Host side of the file: compile_half_cheetah (what mj_loadXML derives from the XML) and the
// launch plumbing.  Arithmetic is fp64 (the reference's); no dense contraction, no tensor cores.
//
// PARITY: unpinned against MuJoCo itself (MuJoCo is not a dependency of this project); pinned
// against the CPU restatement of the same pipeline (tests/ only).  See DESIGN.md section 3.
#include "mujoco.cuh"
#include "mujoco_model.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

namespace epb {

namespace {

using hcm::NV; using hcm::NB; using hcm::NG; using hcm::NU;
using hcm::MINVAL; using hcm::MINIMP; using hcm::MAXIMP;
using hcm::HcModel; using hcm::LegModel;
constexpr int MAXROW = 6 + 3 * 16;  // 6 limits + 16 contacts x 3 merged pyramid rows
constexpr int kStateReals = 32;     // qpos[9] qvel[9] warm[9] norm_saved norm_has pad[3]
constexpr int kWarps = 4;           // envs per CTA

__constant__ HcModel cm;

struct HcParams {
  int frame_skip;
  double ctrl_cost_weight, forward_reward_weight, reset_noise_scale;
};

// ------------------------------------------------------------------ host: model compile
void capsule_inertia(double r, double h, double density, double* mass, double* itrans) {
  double height = 2 * h;
  double mc = density * M_PI * r * r * height;
  double ms = density * 4.0 / 3.0 * M_PI * r * r * r;
  *mass = mc + ms;
  *itrans = mc * (3 * r * r + height * height) / 12.0 +
            ms * (0.4 * r * r + 0.375 * r * height + 0.25 * height * height);
}

// dense Cholesky helpers for the one-time constants (host)
bool host_chol(const double* A, double* L) {
  memcpy(L, A, sizeof(double) * NV * NV);
  for (int j = 0; j < NV; ++j) {
    double d = L[j * NV + j];
    for (int k = 0; k < j; ++k) d -= L[j * NV + k] * L[j * NV + k];
    if (d <= 0) return false;
    d = std::sqrt(d);
    L[j * NV + j] = d;
    for (int i = j + 1; i < NV; ++i) {
      double s = L[i * NV + j];
      for (int k = 0; k < j; ++k) s -= L[i * NV + k] * L[j * NV + k];
      L[i * NV + j] = s / d;
    }
  }
  return true;
}
void host_solve(const double* L, const double* b, double* x) {
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

// What mj_loadXML's compiler does for half_cheetah_envpool.xml (lines cited there):
// geom frames, capsule masses/inertias at density 1000 rescaled to settotalmass=14, body
// CoM / planar inertia, default-class joint parameters, and mj_setConst's inverse weights
// at qpos0.
void compile_half_cheetah(HcModel* m) {
  memset(m, 0, sizeof(*m));
  const int parent[NB] = {-1, 0, 1, 2, 0, 4, 5};
  const double bpos[NB][2] = {{0, 0.7},  {-0.5, 0},      {0.16, -0.25}, {-0.28, -0.14},
                              {0.5, 0},  {-0.14, -0.24}, {0.13, -0.18}};  // xml:71-97
  for (int b = 0; b < NB; ++b) {
    m->parent[b] = parent[b];
    m->bposx[b] = bpos[b][0];
    m->bposz[b] = bpos[b][1];
    int chain[4], n = 0;
    for (int a = b; a >= 0; a = parent[a]) chain[n++] = a + 2;  // body a's hinge dof
    m->chain_len[b] = n;
    m->depth[b] = n - 1;
    for (int k = 0; k < n; ++k) {
      m->chain[b][k] = chain[n - 1 - k];
      m->chainmask[b] |= 1 << chain[k];
    }
  }
  const double damp[6] = {6, 4.5, 3, 4.5, 3, 1.5};
  const double stiff[6] = {240, 180, 120, 180, 120, 60};
  const double range[6][2] = {{-.52, 1.05}, {-.785, .785}, {-.4, .785},
                              {-1, .7},     {-1.2, .87},   {-.5, .5}};  // xml:79-97
  const double gear[NU] = {120, 90, 60, 120, 60, 30};                  // xml:105-110
  for (int j = 0; j < 6; ++j) {
    m->armature[3 + j] = 0.1;  // default class, xml:54
    m->damping[3 + j] = damp[j];
    m->stiffness[3 + j] = stiff[j];
    m->rlo[3 + j] = range[j][0];
    m->rhi[3 + j] = range[j][1];
    m->gear[j] = gear[j];
  }
  m->grad = 0.046;
  struct G { int body; double px, pz, angle, half; bool fromto; };
  const G geoms[NG] = {{0, 0, 0, 0, 0.5, true},           {0, 0.6, 0.1, 0.87, 0.15, false},
                       {1, 0.1, -0.13, -3.8, 0.145, false}, {2, -0.14, -0.07, -2.03, 0.15, false},
                       {3, 0.03, -0.097, -0.27, 0.094, false}, {4, -0.07, -0.12, 0.52, 0.133, false},
                       {5, 0.065, -0.09, -0.6, 0.106, false},  {6, 0.045, -0.07, -0.6, 0.07, false}};
  double gm[NG], gi[NG], total = 0;
  for (int g = 0; g < NG; ++g) {
    m->gbody[g] = geoms[g].body;
    m->gposx[g] = geoms[g].px;
    m->gposz[g] = geoms[g].pz;
    // capsule axis = geom z-axis; axisangle about +y by a: (sin a, cos a) in (x, z);
    // the torso capsule is given by fromto along +x
    m->gaxx[g] = geoms[g].fromto ? 1.0 : std::sin(geoms[g].angle);
    m->gaxz[g] = geoms[g].fromto ? 0.0 : std::cos(geoms[g].angle);
    m->ghalf[g] = geoms[g].half;
    capsule_inertia(m->grad, m->ghalf[g], 1000.0, &gm[g], &gi[g]);
    total += gm[g];
  }
  for (int b = 0; b < NB; ++b) {
    double mb = 0, cx = 0, cz = 0;
    for (int g = 0; g < NG; ++g)
      if (m->gbody[g] == b) {
        mb += gm[g];
        cx += gm[g] * m->gposx[g];
        cz += gm[g] * m->gposz[g];
      }
    cx /= mb;
    cz /= mb;
    double iyy = 0;
    for (int g = 0; g < NG; ++g)
      if (m->gbody[g] == b) {
        double dx = m->gposx[g] - cx, dz = m->gposz[g] - cz;
        iyy += gi[g] + gm[g] * (dx * dx + dz * dz);
      }
    double scale = 14.0 / total;  // settotalmass="14", xml:52
    m->mass[b] = mb * scale;
    m->comx[b] = cx;
    m->comz[b] = cz;
    m->iyy[b] = iyy * scale;
  }
  m->timestep = 0.01;  // xml:59
  m->gravity = -9.81;
  m->mu = 0.4;         // xml:55 (both geoms of every pair carry the default friction)
  m->solref[0] = 0.02; m->solref[1] = 1;
  m->solimp[0] = 0.0; m->solimp[1] = 0.8; m->solimp[2] = 0.01;
  m->solref_limit[0] = 0.02; m->solref_limit[1] = 1;
  m->solimp_limit[0] = 0.0; m->solimp_limit[1] = 0.8; m->solimp_limit[2] = 0.03;
  m->tolerance = 1e-8;  // MuJoCo defaults: Newton, 100 iterations, 50 line-search iterations
  m->max_iter = 100;
  m->ls_iter = 50;
  // mj_setConst at qpos0 = 0: M0, its inverse, dof/body inverse weights, mean inertia
  double org[NB][2], com[NB][2];
  for (int b = 0; b < NB; ++b) {
    int p = m->parent[b];
    org[b][0] = (p < 0 ? 0 : org[p][0]) + m->bposx[b];
    org[b][1] = (p < 0 ? 0 : org[p][1]) + m->bposz[b];
    com[b][0] = org[b][0] + m->comx[b];
    com[b][1] = org[b][1] + m->comz[b];
  }
  double JBx[NB][NV] = {}, JBz[NB][NV] = {}, JBr[NB][NV] = {};
  for (int b = 0; b < NB; ++b) {
    JBx[b][0] = 1;
    JBz[b][1] = 1;
    for (int a = b; a >= 0; a = m->parent[a]) {
      JBx[b][a + 2] = com[b][1] - org[a][1];
      JBz[b][a + 2] = -(com[b][0] - org[a][0]);
      JBr[b][a + 2] = 1;
    }
  }
  double M[NV * NV] = {}, L[NV * NV], Minv[NV * NV];
  for (int b = 0; b < NB; ++b)
    for (int i = 0; i < NV; ++i)
      for (int j = 0; j < NV; ++j)
        M[i * NV + j] += m->mass[b] * (JBx[b][i] * JBx[b][j] + JBz[b][i] * JBz[b][j]) +
                         m->iyy[b] * JBr[b][i] * JBr[b][j];
  for (int i = 0; i < NV; ++i) M[i * NV + i] += m->armature[i];
  host_chol(M, L);
  for (int j = 0; j < NV; ++j) {
    double e[NV] = {}, x[NV];
    e[j] = 1;
    host_solve(L, e, x);
    for (int i = 0; i < NV; ++i) Minv[i * NV + j] = x[i];
  }
  double tr = 0;
  for (int i = 0; i < NV; ++i) {
    m->dof_invweight0[i] = Minv[i * NV + i];
    tr += M[i * NV + i];
  }
  m->meaninertia = tr / NV;
  for (int b = 0; b < NB; ++b) {
    double axx = 0, azz = 0;
    for (int i = 0; i < NV; ++i)
      for (int j = 0; j < NV; ++j) {
        axx += JBx[b][i] * Minv[i * NV + j] * JBx[b][j];
        azz += JBz[b][i] * Minv[i * NV + j] * JBz[b][j];
      }
    m->body_invw_tran[b] = (axx + azz) / 3.0;  // the y row is identically zero (planar)
  }
  hcm::fill_impedance_constants(m);
}

// ---------------------------------------------------------------- device: per-warp memory
struct WarpMem {
  double q[NV], v[NV], warm[NV], ctrl[NU];
  double org[NB][2], cs[NB][2], com[NB][2], acom[NB][2], omega[NB], aorg[NB][2];
  double JBx[NB][NV], JBz[NB][NV];
  double M[NV * NV], L[NV * NV];
  double fs[NV], as[NV], a[NV], Ma[NV], grad[NV], srch[NV], Mv[NV], fc[NV], tmp[NV];
  double J[MAXROW][NV];
  double D[MAXROW], aref[MAXROW], jar[MAXROW], Jv[MAXROW];
};

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// L <- chol(L) in place (lower triangle), warp-cooperative right-looking factorisation
__device__ __forceinline__ void warp_chol(double* L, int lane) {
  for (int j = 0; j < NV; ++j) {
    double d = sqrt(L[j * NV + j]);
    __syncwarp();
    if (lane == j) L[j * NV + j] = d;
    if (lane > j && lane < NV) L[lane * NV + j] /= d;
    __syncwarp();
    // trailing update: pairs (i, k) with j < k <= i < NV
    for (int t = lane; t < 36; t += 32) {
      // decode t -> (i, k) over the strict+diag lower triangle of an 8x8 (rows 1..8)
      int i = 1, rem = t;
      while (rem >= i) { rem -= i; ++i; }  // row i (1..8) has i entries k = 1..i
      int k = rem + 1;
      if (k > j && i > j) L[i * NV + k] -= L[i * NV + j] * L[k * NV + j];
    }
    __syncwarp();
  }
}

// solve L L^T x = b; x may alias b.  Column-oriented substitutions, lanes own entries.
__device__ __forceinline__ void warp_chol_solve(const double* L, double* x, int lane) {
  for (int j = 0; j < NV; ++j) {
    if (lane == j) x[j] /= L[j * NV + j];
    __syncwarp();
    if (lane > j && lane < NV) x[lane] -= L[lane * NV + j] * x[j];
    __syncwarp();
  }
  for (int j = NV - 1; j >= 0; --j) {
    if (lane == j) x[j] /= L[j * NV + j];
    __syncwarp();
    if (lane < j) x[lane] -= L[j * NV + lane] * x[j];
    __syncwarp();
  }
}

__device__ __noinline__ void impedance(const double* solref, const double* solimp,
                                          double pos, double& imp, double& K, double& B) {
  double dmin = fmin(MAXIMP, fmax(MINIMP, solimp[0]));
  double dmax = fmin(MAXIMP, fmax(MINIMP, solimp[1]));
  double x = fabs(pos) / solimp[2];
  if (x >= 1) {
    imp = dmax;
  } else if (x <= 0) {
    imp = dmin;
  } else {
    // midpoint 0.5, power 2 (MuJoCo defaults for the unspecified solimp entries)
    double y = x <= 0.5 ? (x * x) / 0.5 : 1 - ((1 - x) * (1 - x)) / 0.5;
    imp = dmin + y * (dmax - dmin);
  }
  K = 1 / fmax(MINVAL, dmax * dmax * solref[0] * solref[0] * solref[1] * solref[1]);
  B = 2 / fmax(MINVAL, dmax * solref[0]);
}

// ------------------------------------------------------------------- one mj_step (warp)
__device__ void hc_substep(WarpMem& w, int lane) {
  // ---- position stage: kinematics ------------------------------------------------------
  if (lane < NB) {
    double th = 0;
    for (int k = 0; k < cm.chain_len[lane]; ++k) th += w.q[cm.chain[lane][k]];
    double s, c;
    sincos(th, &s, &c);
    w.cs[lane][0] = c;
    w.cs[lane][1] = s;
    double om = 0;
    for (int k = 0; k < cm.chain_len[lane]; ++k) om += w.v[cm.chain[lane][k]];
    w.omega[lane] = om;
  }
  __syncwarp();
  for (int d = 0; d < 4; ++d) {
    if (lane < NB && cm.depth[lane] == d) {
      int p = cm.parent[lane];
      if (p < 0) {
        w.org[lane][0] = cm.bposx[lane] + w.q[0];
        w.org[lane][1] = cm.bposz[lane] + w.q[1];
        w.aorg[lane][0] = 0;
        w.aorg[lane][1] = 0;
      } else {
        double c = w.cs[p][0], s = w.cs[p][1];
        double rx = c * cm.bposx[lane] + s * cm.bposz[lane];
        double rz = -s * cm.bposx[lane] + c * cm.bposz[lane];
        w.org[lane][0] = w.org[p][0] + rx;
        w.org[lane][1] = w.org[p][1] + rz;
        double op2 = w.omega[p] * w.omega[p];
        w.aorg[lane][0] = w.aorg[p][0] - op2 * rx;
        w.aorg[lane][1] = w.aorg[p][1] - op2 * rz;
      }
    }
    __syncwarp();
  }
  if (lane < NB) {
    const int b = lane;
    double c = w.cs[b][0], s = w.cs[b][1];
    double rx = c * cm.comx[b] + s * cm.comz[b];
    double rz = -s * cm.comx[b] + c * cm.comz[b];
    double cx = w.org[b][0] + rx, cz = w.org[b][1] + rz;
    w.com[b][0] = cx;
    w.com[b][1] = cz;
    double o2 = w.omega[b] * w.omega[b];
    w.acom[b][0] = w.aorg[b][0] - o2 * rx;
    w.acom[b][1] = w.aorg[b][1] - o2 * rz - cm.gravity;  // a - g
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      w.JBx[b][i] = 0;
      w.JBz[b][i] = 0;
    }
    w.JBx[b][0] = 1;
    w.JBz[b][1] = 1;
    for (int a = b; a >= 0; a = cm.parent[a]) {
      w.JBx[b][a + 2] = cz - w.org[a][1];
      w.JBz[b][a + 2] = -(cx - w.org[a][0]);
    }
  }
  __syncwarp();
  // ---- joint-space inertia M (lower triangle, mirrored) -------------------------------
  for (int t = lane; t < 45; t += 32) {
    int i = 0, rem = t;
    while (rem > i) { rem -= i + 1; ++i; }
    int j = rem;  // j <= i
    double acc = 0;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      // rotational Jacobian entries are 1 on the body's hinge chain
      double ri = (double)((cm.chainmask[b] >> i) & 1);
      double rj = (double)((cm.chainmask[b] >> j) & 1);
      acc += cm.mass[b] * (w.JBx[b][i] * w.JBx[b][j] + w.JBz[b][i] * w.JBz[b][j]) +
             cm.iyy[b] * ri * rj;
    }
    if (i == j) acc += cm.armature[i];
    w.M[i * NV + j] = acc;
    w.M[j * NV + i] = acc;
  }
  // ---- velocity stage: bias, passive; actuation; qfrc_smooth ---------------------------
  if (lane < NV) {
    const int i = lane;
    double bias = 0;
#pragma unroll
    for (int b = 0; b < NB; ++b)
      bias += cm.mass[b] * (w.JBx[b][i] * w.acom[b][0] + w.JBz[b][i] * w.acom[b][1]);
    double passive = -cm.stiffness[i] * w.q[i] - cm.damping[i] * w.v[i];
    double act = 0;
    if (i >= 3) {
      double c = w.ctrl[i - 3];
      c = c < -1 ? -1 : (c > 1 ? 1 : c);  // ctrllimited, ctrlrange -1 1
      act = cm.gear[i - 3] * c;
    }
    double f = passive - bias + act;
    w.fs[i] = f;
    w.as[i] = f;
  }
  __syncwarp();
  for (int t = lane; t < NV * NV; t += 32) w.L[t] = w.M[t];
  __syncwarp();
  warp_chol(w.L, lane);
  warp_chol_solve(w.L, w.as, lane);  // qacc_smooth
  // ---- collision + constraint rows ------------------------------------------------------
  bool lim = false, con = false;
  double ldist = 0, lsign = 0;
  int ldof = 0;
  double pJx[NV], pJz[NV], cdist = 0;
  int cbody = 0;
  if (lane >= 16 && lane < 22) {  // joint limits, mj_instantiateLimit
    ldof = 3 + (lane - 16);
    double qv = w.q[ldof];
    double dlo = qv - cm.rlo[ldof], dhi = cm.rhi[ldof] - qv;
    if (dlo < 0) {
      lim = true; ldist = dlo; lsign = 1;
    } else if (dhi < 0) {
      lim = true; ldist = dhi; lsign = -1;
    }
  }
  if (lane < 16) {  // floor plane vs capsule end spheres (mjc_PlaneCapsule), margin 0
    int g = lane >> 1;
    double end = (lane & 1) ? -1.0 : 1.0;
    cbody = cm.gbody[g];
    double c = w.cs[cbody][0], s = w.cs[cbody][1];
    double gx = w.org[cbody][0] + c * cm.gposx[g] + s * cm.gposz[g];
    double gz = w.org[cbody][1] - s * cm.gposx[g] + c * cm.gposz[g];
    double ax = c * cm.gaxx[g] + s * cm.gaxz[g];
    double az = -s * cm.gaxx[g] + c * cm.gaxz[g];
    double px = gx + end * cm.ghalf[g] * ax, pz = gz + end * cm.ghalf[g] * az;
    if (!(pz > cm.grad)) {
      con = true;
      cdist = pz - cm.grad;
      double cpz = pz - (cm.grad + cdist / 2);  // sphere centre - n (radius + dist/2)
#pragma unroll
      for (int i = 0; i < NV; ++i) pJx[i] = pJz[i] = 0;
      pJx[0] = 1;
      pJz[1] = 1;
      for (int a = cbody; a >= 0; a = cm.parent[a]) {
        pJx[a + 2] = cpz - w.org[a][1];
        pJz[a + 2] = -(px - w.org[a][0]);
      }
    }
  }
  const unsigned lmask = __ballot_sync(0xffffffffu, lim);
  const unsigned cmask = __ballot_sync(0xffffffffu, con);
  const int nlim = __popc(lmask), ncon = __popc(cmask);
  const int nrow = nlim + 3 * ncon;
  const unsigned below = (1u << lane) - 1u;
  if (lim) {
    int r = __popc(lmask & below);
    double imp, K, B;
    impedance(cm.solref_limit, cm.solimp_limit, ldist, imp, K, B);
    double R = fmax(MINVAL, (1 - imp) * cm.dof_invweight0[ldof] / imp);
#pragma unroll
    for (int i = 0; i < NV; ++i) w.J[r][i] = 0;
    w.J[r][ldof] = lsign;
    w.D[r] = 1 / R;
    w.aref[r] = -B * (lsign * w.v[ldof]) - K * imp * ldist;
  }
  if (con) {
    int r = nlim + 3 * __popc(cmask & below);
    double velx = 0, velz = 0;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      velx += pJx[i] * w.v[i];
      velz += pJz[i] * w.v[i];
    }
    double imp, K, B;
    impedance(cm.solref, cm.solimp, cdist, imp, K, B);
    // mj_diagApprox (pyramidal): tran + mu^2 tran; R of every edge = 2 mu^2 R(first edge)
    double tran = cm.body_invw_tran[cbody];
    double dA = tran + cm.mu * cm.mu * tran;
    double R = fmax(MINVAL, (1 - imp) * dA / imp) * (2 * cm.mu * cm.mu);
    double D = 1 / R, kip = K * imp * cdist;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      w.J[r][i] = pJz[i] + cm.mu * pJx[i];
      w.J[r + 1][i] = pJz[i] - cm.mu * pJx[i];
      w.J[r + 2][i] = pJz[i];
    }
    w.D[r] = D;
    w.D[r + 1] = D;
    w.D[r + 2] = 2 * D;  // the two identical (n +- mu t_y) edges merged into one row
    w.aref[r] = -B * (velz + cm.mu * velx) - kip;
    w.aref[r + 1] = -B * (velz - cm.mu * velx) - kip;
    w.aref[r + 2] = -B * velz - kip;
  }
  __syncwarp();
  // ---- constraint solve -------------------------------------------------------------------
  if (nrow == 0) {
    if (lane < NV) {
      w.a[lane] = w.as[lane];
      w.fc[lane] = 0;
    }
    __syncwarp();
  } else {
    // warmstart: keep qacc_warmstart only if its cost beats the cost at qacc_smooth
    double cw = 0, cs = 0;
    for (int r = lane; r < nrow; r += 32) {
      double sw = -w.aref[r], ss = -w.aref[r];
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        sw += w.J[r][i] * w.warm[i];
        ss += w.J[r][i] * w.as[i];
      }
      if (sw < 0) cw += 0.5 * w.D[r] * sw * sw;
      if (ss < 0) cs += 0.5 * w.D[r] * ss * ss;
    }
    if (lane < NV) {
      double ma = 0;
#pragma unroll
      for (int k = 0; k < NV; ++k) ma += w.M[lane * NV + k] * w.warm[k];
      cw += 0.5 * (ma - w.fs[lane]) * (w.warm[lane] - w.as[lane]);
    }
    cw = warp_sum(cw);
    cs = warp_sum(cs);
    if (lane < NV) w.a[lane] = cw > cs ? w.as[lane] : w.warm[lane];
    __syncwarp();
    const double scale = 1.0 / (cm.meaninertia * NV);
    double cost = 0;
    for (int iter = 0; iter <= cm.max_iter; ++iter) {
      // constraint update at the current point
      if (lane < NV) {
        double ma = 0;
#pragma unroll
        for (int k = 0; k < NV; ++k) ma += w.M[lane * NV + k] * w.a[k];
        w.Ma[lane] = ma;
      }
      double part = 0;
      for (int r = lane; r < nrow; r += 32) {
        double s = -w.aref[r];
#pragma unroll
        for (int i = 0; i < NV; ++i) s += w.J[r][i] * w.a[i];
        w.jar[r] = s;
        if (s < 0) part += 0.5 * w.D[r] * s * s;
      }
      __syncwarp();
      double g2 = 0;
      if (lane < NV) {
        double fc = 0;
        for (int r = 0; r < nrow; ++r) {
          double s = w.jar[r];
          if (s < 0) fc += w.J[r][lane] * (-w.D[r] * s);
        }
        w.fc[lane] = fc;
        double g = w.Ma[lane] - w.fs[lane] - fc;
        w.grad[lane] = g;
        g2 = g * g;
        part += 0.5 * (w.Ma[lane] - w.fs[lane]) * (w.a[lane] - w.as[lane]);
      }
      const double newcost = warp_sum(part);
      const double gnorm = sqrt(warp_sum(g2));
      if (iter > 0) {
        if (scale * (cost - newcost) < cm.tolerance || scale * gnorm < cm.tolerance) break;
      } else if (scale * gnorm < cm.tolerance) {
        break;
      }
      cost = newcost;
      if (iter == cm.max_iter) break;
      // Newton direction: H = M + J^T D_active J
      for (int t = lane; t < 45; t += 32) {
        int i = 0, rem = t;
        while (rem > i) { rem -= i + 1; ++i; }
        int j = rem;
        double h = w.M[i * NV + j];
        for (int r = 0; r < nrow; ++r)
          if (w.jar[r] < 0) h += w.D[r] * w.J[r][i] * w.J[r][j];
        w.L[i * NV + j] = h;
      }
      if (lane < NV) w.srch[lane] = w.grad[lane];
      __syncwarp();
      warp_chol(w.L, lane);
      warp_chol_solve(w.L, w.srch, lane);
      if (lane < NV) w.srch[lane] = -w.srch[lane];
      __syncwarp();
      // exact line search: safeguarded Newton on phi'(alpha)
      double q1 = 0, q2 = 0;
      if (lane < NV) {
        double mv = 0;
#pragma unroll
        for (int k = 0; k < NV; ++k) mv += w.M[lane * NV + k] * w.srch[k];
        q1 = w.srch[lane] * (w.Ma[lane] - w.fs[lane]);
        q2 = w.srch[lane] * mv;
      }
      for (int r = lane; r < nrow; r += 32) {
        double s = 0;
#pragma unroll
        for (int i = 0; i < NV; ++i) s += w.J[r][i] * w.srch[i];
        w.Jv[r] = s;
      }
      q1 = warp_sum(q1);
      q2 = warp_sum(q2);
      __syncwarp();
      double sn2 = (lane < NV) ? w.srch[lane] * w.srch[lane] : 0.0;
      const double gtol = cm.tolerance * 0.01 * sqrt(warp_sum(sn2)) / scale;
      double lo = 0, hi = INFINITY, alpha = 0;
      for (int k = 0; k < cm.ls_iter; ++k) {
        double d1 = 0, d2 = 0;
        for (int r = lane; r < nrow; r += 32) {
          double x = w.jar[r] + alpha * w.Jv[r];
          if (x < 0) {
            d1 += w.D[r] * x * w.Jv[r];
            d2 += w.D[r] * w.Jv[r] * w.Jv[r];
          }
        }
        d1 = warp_sum(d1) + (q1 + alpha * q2);
        d2 = warp_sum(d2) + q2;
        if (fabs(d1) < gtol) break;
        if (d1 < 0) lo = alpha; else hi = alpha;
        double next = alpha - d1 / d2;
        if (!(next > lo && next < hi)) next = isinf(hi) ? 2 * alpha + 1 : 0.5 * (lo + hi);
        if (next == alpha) break;
        alpha = next;
      }
      if (alpha == 0) break;
      if (lane < NV) w.a[lane] += alpha * w.srch[lane];
      __syncwarp();
    }
  }
  // ---- mj_Euler with implicit joint damping -------------------------------------------------
  for (int t = lane; t < NV * NV; t += 32) {
    int i = t / NV, j = t - i * NV;
    w.L[t] = w.M[t] + (i == j ? cm.timestep * cm.damping[i] : 0.0);
  }
  if (lane < NV) w.tmp[lane] = w.fs[lane] + w.fc[lane];
  __syncwarp();
  warp_chol(w.L, lane);
  warp_chol_solve(w.L, w.tmp, lane);
  if (lane < NV) {
    double vnew = w.v[lane] + cm.timestep * w.tmp[lane];
    w.v[lane] = vnew;
    w.q[lane] += cm.timestep * vnew;
    w.warm[lane] = w.a[lane];  // mj_advance: qacc_warmstart <- solver qacc
  }
  __syncwarp();
}

// std::normal_distribution<double> (libstdc++ 13 bits/random.tcc:1811-1844)
__device__ double hc_normal(Mt& rng, double& saved, bool& has_saved, double mean, double sd) {
  double ret;
  if (has_saved) {
    has_saved = false;
    ret = saved;
  } else {
    double x, y, r2;
    do {
      uint32_t d[4];
      rng.next_batch<4>(d);
      x = __dsub_rn(__dmul_rn(2.0, Mt::canonical_from(d[0], d[1])), 1.0);
      y = __dsub_rn(__dmul_rn(2.0, Mt::canonical_from(d[2], d[3])), 1.0);
      r2 = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    } while (r2 > 1.0 || r2 == 0.0);
    double mult = sqrt(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2));
    saved = __dmul_rn(x, mult);
    has_saved = true;
    ret = __dmul_rn(y, mult);
  }
  return __dadd_rn(__dmul_rn(ret, sd), mean);
}

// One launch = T sync steps (T = 1 for the single-step API) of `n` batch rows; warp = row.
__global__ void __launch_bounds__(kWarps * 32)
hc_kernel(StateView sv, OutView ov, HcParams prm, const double* __restrict__ action,
          const int32_t* __restrict__ env_ids, int n, int force_reset, int T) {
  __shared__ WarpMem wm[kWarps];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int row = blockIdx.x * kWarps + wid;
  if (row >= n) return;  // whole warp exits together
  WarpMem& w = wm[wid];
  const int eid = env_ids ? env_ids[row] : row;
  double* st = static_cast<double*>(sv.rstate) + eid;  // SoA: real k of env e at k*N + e
  const int64_t N = sv.n_envs;
  int flags = sv.flags[eid];
  if (lane < NV) {
    w.q[lane] = st[lane * N];
    w.v[lane] = st[(NV + lane) * N];
    w.warm[lane] = st[(2 * NV + lane) * N];
  }
  __syncwarp();
  for (int t = 0; t < T; ++t) {
    const int64_t orow = (int64_t)t * ov.t_stride_rows + row;
    int done = flags & 1, cur = flags >> 1;
    const bool reset = force_reset || done;
    double xv = 0, ctrl_cost = 0, x_after = 0;
    float reward = 0.0f;
    if (reset) {
      // HalfCheetahEnv::Reset + MujocoReset + MujocoResetModel (half_cheetah.h:105-134,
      // mujoco_env.h:126-131): mj_resetData, qpos = init + U(-s, s), qvel = init + N(0, s)
      cur = 0;
      done = 0;
      if (lane == 0) {
        Mt rng(sv, eid);
        double saved = st[27 * N];
        bool has = st[28 * N] != 0.0;
        double u[NV];
        rng.uniform_real_batch<NV>(-prm.reset_noise_scale, prm.reset_noise_scale, u);
        for (int i = 0; i < NV; ++i) w.q[i] = 0.0 + u[i];
        for (int i = 0; i < NV; ++i)
          w.v[i] = 0.0 + hc_normal(rng, saved, has, 0.0, prm.reset_noise_scale);
        for (int i = 0; i < NV; ++i) w.warm[i] = 0.0;
        rng.save(sv, eid);
        st[27 * N] = saved;
        st[28 * N] = has ? 1.0 : 0.0;
      }
      __syncwarp();
    } else {
      ++cur;
      const double* act = action + ((int64_t)t * n + row) * NU;
      if (lane < NU) w.ctrl[lane] = act[lane];
      __syncwarp();
      const double x_before = w.q[0];
      for (int k = 0; k < prm.frame_skip; ++k) hc_substep(w, lane);
      x_after = w.q[0];
      // env-layer algebra (half_cheetah.h:147-160) with explicit _rn ops: never FMA-contracted,
      // so reward / infos are the x86-64 double results given the same qpos, ctrl
      for (int k = 0; k < NU; ++k)
        ctrl_cost = __dadd_rn(ctrl_cost, __dmul_rn(__dmul_rn(prm.ctrl_cost_weight, w.ctrl[k]), w.ctrl[k]));
      const double dt = prm.frame_skip * cm.timestep;
      xv = (x_after - x_before) / dt;
      reward = (float)__dsub_rn(__dmul_rn(xv, prm.forward_reward_weight), ctrl_cost);
      done = (cur >= sv.max_steps);
    }
    flags = (cur << 1) | done;
    if (lane == 0) {
      write_common(ov, orow, eid + sv.env_id_offset, cur, done, reward, sv.max_steps);
      // infos (half_cheetah.h:178-181); on reset WriteState gets literal zeros
      if (ov.env[1]) static_cast<double*>(ov.env[1])[orow] = __dmul_rn(xv, prm.forward_reward_weight);
      if (ov.env[2]) static_cast<double*>(ov.env[2])[orow] = -ctrl_cost;
      if (ov.env[3]) static_cast<double*>(ov.env[3])[orow] = x_after;
      if (ov.env[4]) static_cast<double*>(ov.env[4])[orow] = xv;
    }
    if (ov.env[0] && lane < 17)  // obs = qpos[1:9] ++ qvel[0:9]
      static_cast<double*>(ov.env[0])[orow * 17 + lane] = lane < 8 ? w.q[lane + 1] : w.v[lane - 8];
    __syncwarp();
  }
  if (lane < NV) {
    st[lane * N] = w.q[lane];
    st[(NV + lane) * N] = w.v[lane];
    st[(2 * NV + lane) * N] = w.warm[lane];
  }
  if (lane == 0) sv.flags[eid] = flags;
}

}  // namespace
}  // namespace epb

#include "mujoco_thread.cuh"

namespace epb {
namespace {

constexpr int kThreadBlock = 64;

// One launch = T sync steps of `n` batch rows; ONE THREAD PER ENV (row).
//
// `lane_shift` (experiment, default 0): only every (1 << lane_shift)-th lane of a warp carries
// an env -- see hc_lane_shift() for why spreading a small batch over more warps does not pay.
__global__ void __launch_bounds__(kThreadBlock)
hc_thread_kernel(StateView sv, OutView ov, HcParams prm, const double* __restrict__ action,
                 const int32_t* __restrict__ env_ids, int n, int force_reset, int T,
                 int lane_shift) {
  const int tid = blockIdx.x * kThreadBlock + threadIdx.x;
  if (tid & ((1 << lane_shift) - 1)) return;
  const int row = tid >> lane_shift;
  if (row >= n) return;
  const int eid = env_ids ? env_ids[row] : row;
  const int64_t N = sv.n_envs;
  double* st = static_cast<double*>(sv.rstate) + eid;
  hct::HcState s;
  hct::Rows e;
  int flags = sv.flags[eid];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    s.q[i] = st[i * N];
    s.v[i] = st[(NV + i) * N];
    s.warm[i] = st[(2 * NV + i) * N];
  }
  for (int t = 0; t < T; ++t) {
    const int64_t orow = (int64_t)t * ov.t_stride_rows + row;
    int done = flags & 1, cur = flags >> 1;
    const bool reset = force_reset || done;
    double xv = 0, ctrl_cost = 0, x_after = 0;
    float reward = 0.0f;
    if (reset) {
      cur = 0;
      done = 0;
      Mt rng(sv, eid);
      double saved = st[27 * N];
      bool has = st[28 * N] != 0.0;
      double u[NV];
      rng.uniform_real_batch<NV>(-prm.reset_noise_scale, prm.reset_noise_scale, u);
#pragma unroll
      for (int i = 0; i < NV; ++i) s.q[i] = 0.0 + u[i];
      for (int i = 0; i < NV; ++i)
        s.v[i] = 0.0 + hc_normal(rng, saved, has, 0.0, prm.reset_noise_scale);
#pragma unroll
      for (int i = 0; i < NV; ++i) s.warm[i] = 0.0;
      rng.save(sv, eid);
      st[27 * N] = saved;
      st[28 * N] = has ? 1.0 : 0.0;
    } else {
      ++cur;
      const double* act = action + ((int64_t)t * n + row) * NU;
#pragma unroll
      for (int k = 0; k < NU; ++k) s.ctrl[k] = act[k];
      const double x_before = s.q[0];
      for (int k = 0; k < prm.frame_skip; ++k) hct::substep(s, e);
      x_after = s.q[0];
#pragma unroll
      // env-layer algebra (half_cheetah.h:147-160) with explicit _rn ops: never FMA-contracted,
      // so reward / infos are the x86-64 double results given the same qpos, ctrl
      for (int k = 0; k < NU; ++k)
        ctrl_cost = __dadd_rn(ctrl_cost, __dmul_rn(__dmul_rn(prm.ctrl_cost_weight, s.ctrl[k]), s.ctrl[k]));
      const double dt = prm.frame_skip * cm.timestep;
      xv = (x_after - x_before) / dt;
      reward = (float)__dsub_rn(__dmul_rn(xv, prm.forward_reward_weight), ctrl_cost);
      done = (cur >= sv.max_steps);
    }
    flags = (cur << 1) | done;
    write_common(ov, orow, eid + sv.env_id_offset, cur, done, reward, sv.max_steps);
    if (ov.env[1]) static_cast<double*>(ov.env[1])[orow] = __dmul_rn(xv, prm.forward_reward_weight);
    if (ov.env[2]) static_cast<double*>(ov.env[2])[orow] = -ctrl_cost;
    if (ov.env[3]) static_cast<double*>(ov.env[3])[orow] = x_after;
    if (ov.env[4]) static_cast<double*>(ov.env[4])[orow] = xv;
    if (ov.env[0]) {
      double* o = static_cast<double*>(ov.env[0]) + orow * 17;
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = s.q[k + 1];
#pragma unroll
      for (int k = 0; k < 9; ++k) o[8 + k] = s.v[k];
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    st[i * N] = s.q[i];
    st[(NV + i) * N] = s.v[i];
    st[(2 * NV + i) * N] = s.warm[i];
  }
  sv.flags[eid] = flags;
}

}  // namespace
}  // namespace epb

#include "mujoco_pair.cuh"

namespace epb {
namespace {

constexpr int kPairBlock = 64;  // threads per CTA = 32 envs
constexpr int kPairKsMin = 9;   // fewest constraint rows per lane ever held in shared memory
static_assert(kPairBlock == HCP_SSTRIDE, "row interleave stride = threads per CTA");

// the two LegModel tables in global memory (written once per process, mjc_pool_create): every
// CTA copies them into shared memory with one coalesced read
__device__ LegModel g_leg_model[2];

// One launch = T sync steps of `n` batch rows; TWO LANES PER ENV (mujoco_pair.cuh): lane
// 2*row is the back leg (and does everything that exists once per env: RNG, reward, the
// common columns), lane 2*row + 1 the front leg.  Dynamic shared memory: the first `ks`
// constraint rows of every lane, interleaved by thread.
//
// 245 registers, no spills: 4 CTAs (8 warps) per SM.  Builds capped at 144 and 128 registers
// (7 / 8 CTAs per SM: fewer waves) were measured and dropped: their spills cost more than the
// extra wave.
__global__ void __launch_bounds__(kPairBlock)
hc_pair_kernel(StateView sv, OutView ov, HcParams prm, const double* __restrict__ action,
               const int32_t* __restrict__ env_ids, int n, int force_reset, int T, int ks) {
  extern __shared__ double srows[];
  __shared__ LegModel lm[2];
  {
    const double* src = reinterpret_cast<const double*>(g_leg_model);
    double* dst = reinterpret_cast<double*>(lm);
    for (int i = threadIdx.x; i < (int)(2 * sizeof(LegModel) / sizeof(double)); i += kPairBlock)
      dst[i] = src[i];
  }
  __syncthreads();
  const int tid = blockIdx.x * kPairBlock + threadIdx.x;
  const int row = tid >> 1, side = tid & 1;
  if (row >= n) return;  // both lanes of a pair leave together
  const int eid = env_ids ? env_ids[row] : row;
  const int64_t N = sv.n_envs;
  double* st = static_cast<double*>(sv.rstate) + eid;
  double ovf[(hcp::MAXR - kPairKsMin) * hcp::NF];
  hcp::Ctx c;
  c.side = side;
  c.pm = 3u << (threadIdx.x & 30);
  c.chan = nullptr;
  c.srow = srows + threadIdx.x;
  c.ks = ks;
  c.ovf = ovf;
  const LegModel& L = lm[side];
  const int l0 = 3 + 3 * side;  // first dof of this lane's leg
  hcp::PairState s;
  int flags = sv.flags[eid];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    s.qr[i] = st[i * N];
    s.vr[i] = st[(NV + i) * N];
    s.wr[i] = st[(2 * NV + i) * N];
    s.ql[i] = st[(l0 + i) * N];
    s.vl[i] = st[(NV + l0 + i) * N];
    s.wl[i] = st[(2 * NV + l0 + i) * N];
  }
  for (int t = 0; t < T; ++t) {
    const int64_t orow = (int64_t)t * ov.t_stride_rows + row;
    int done = flags & 1, cur = flags >> 1;
    const bool reset = force_reset || done;
    double xv = 0, ctrl_cost = 0, x_after = 0;
    float reward = 0.0f;
    if (reset) {
      // HalfCheetahEnv::Reset (half_cheetah.h:105-134): the back-leg lane draws, both keep
      // their part
      cur = 0;
      done = 0;
      double q9[NV], v9[NV];
#pragma unroll
      for (int i = 0; i < NV; ++i) q9[i] = v9[i] = 0.0;
      if (side == 0) {
        Mt rng(sv, eid);
        double saved = st[27 * N];
        bool has = st[28 * N] != 0.0;
        rng.uniform_real_batch<NV>(-prm.reset_noise_scale, prm.reset_noise_scale, q9);
#pragma unroll
        for (int i = 0; i < NV; ++i) q9[i] = 0.0 + q9[i];
        for (int i = 0; i < NV; ++i)
          v9[i] = 0.0 + hc_normal(rng, saved, has, 0.0, prm.reset_noise_scale);
        rng.save(sv, eid);
        st[27 * N] = saved;
        st[28 * N] = has ? 1.0 : 0.0;
      }
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const double qo = hcp::xch(c, q9[i]), vo = hcp::xch(c, v9[i]);
        if (side) { q9[i] = qo; v9[i] = vo; }
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        s.qr[i] = q9[i];
        s.vr[i] = v9[i];
        s.ql[i] = side ? q9[6 + i] : q9[3 + i];
        s.vl[i] = side ? v9[6 + i] : v9[3 + i];
        s.wr[i] = 0.0;
        s.wl[i] = 0.0;
      }
    } else {
      ++cur;
      const double* act = action + ((int64_t)t * n + row) * NU;
      double a6[NU];
#pragma unroll
      for (int k = 0; k < NU; ++k) a6[k] = act[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) s.ctrl[k] = side ? a6[3 + k] : a6[k];
      const double x_before = s.qr[0];
      for (int k = 0; k < prm.frame_skip; ++k) hcp::pair_substep(c, cm, L, s);
      x_after = s.qr[0];
      // env-layer algebra (half_cheetah.h:147-160) with explicit _rn ops: never FMA-contracted
#pragma unroll
      for (int k = 0; k < NU; ++k)
        ctrl_cost = __dadd_rn(ctrl_cost, __dmul_rn(__dmul_rn(prm.ctrl_cost_weight, a6[k]), a6[k]));
      const double dt = prm.frame_skip * cm.timestep;
      xv = (x_after - x_before) / dt;
      reward = (float)__dsub_rn(__dmul_rn(xv, prm.forward_reward_weight), ctrl_cost);
      done = (cur >= sv.max_steps);
    }
    flags = (cur << 1) | done;
    double* o = ov.env[0] ? static_cast<double*>(ov.env[0]) + orow * 17 : nullptr;
    if (side == 0) {
      write_common(ov, orow, eid + sv.env_id_offset, cur, done, reward, sv.max_steps);
      if (ov.env[1]) static_cast<double*>(ov.env[1])[orow] = __dmul_rn(xv, prm.forward_reward_weight);
      if (ov.env[2]) static_cast<double*>(ov.env[2])[orow] = -ctrl_cost;
      if (ov.env[3]) static_cast<double*>(ov.env[3])[orow] = x_after;
      if (ov.env[4]) static_cast<double*>(ov.env[4])[orow] = xv;
      if (o) {
        o[0] = s.qr[1]; o[1] = s.qr[2];
#pragma unroll
        for (int k = 0; k < 3; ++k) { o[2 + k] = s.ql[k]; o[8 + k] = s.vr[k]; o[11 + k] = s.vl[k]; }
      }
    } else if (o) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { o[5 + k] = s.ql[k]; o[14 + k] = s.vl[k]; }
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (side == 0) {
      st[i * N] = s.qr[i];
      st[(NV + i) * N] = s.vr[i];
      st[(2 * NV + i) * N] = s.wr[i];
    }
    st[(l0 + i) * N] = s.ql[i];
    st[(NV + l0 + i) * N] = s.vl[i];
    st[(2 * NV + l0 + i) * N] = s.wl[i];
  }
  if (side == 0) sv.flags[eid] = flags;
}

}  // namespace

struct MjcPool {
  HcParams prm;
  int num_envs;
  int variant;  // 0 = lane pair per env (default), 1 = thread per env, 2 = warp per env
                // (ENVPOOL_B200_HC_KERNEL=pair|thread|warp)
};

MjcPool* mjc_pool_create(int num_envs, int precision, int frame_skip, double ctrl_cost_weight,
                         double forward_reward_weight, double reset_noise_scale) {
  (void)precision;  // HalfCheetah always computes in fp64 (DESIGN.md)
  static HcModel host_model;
  compile_half_cheetah(&host_model);
  if (cudaMemcpyToSymbol(cm, &host_model, sizeof(HcModel)) != cudaSuccess) return nullptr;
  MjcPool* m = new MjcPool();
  m->num_envs = num_envs;
  m->prm.frame_skip = frame_skip;
  m->prm.ctrl_cost_weight = ctrl_cost_weight;
  m->prm.forward_reward_weight = forward_reward_weight;
  m->prm.reset_noise_scale = reset_noise_scale;
  const char* v = getenv("ENVPOOL_B200_HC_KERNEL");
  m->variant = 0;
  if (v && std::string(v) == "thread") m->variant = 1;
  if (v && std::string(v) == "warp") m->variant = 2;
  if (m->variant == 0) {
    LegModel legs[2];
    hcm::leg_model_of(host_model, 0, &legs[0]);
    hcm::leg_model_of(host_model, 1, &legs[1]);
    const int smem_max = hcp::MAXR * hcp::NF * kPairBlock * (int)sizeof(double);
    if (cudaMemcpyToSymbol(g_leg_model, legs, sizeof(legs)) != cudaSuccess ||
        cudaFuncSetAttribute(hc_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             smem_max) != cudaSuccess) {
      delete m;
      return nullptr;
    }
  }
  return m;
}
void mjc_pool_destroy(MjcPool* m) { delete m; }
// The compiled model as a flat blob (hcm::HcModel): host-only, for the CPU tests that run the
// pair-lane algorithm on host threads.
int64_t mjc_model_blob(void* dst, int64_t cap) {
  if (dst && cap >= (int64_t)sizeof(HcModel)) {
    HcModel tmp;
    compile_half_cheetah(&tmp);
    memcpy(dst, &tmp, sizeof(HcModel));
  }
  return (int64_t)sizeof(HcModel);
}
int mjc_state_reals(const MjcPool*) { return kStateReals; }

// Lane spreading of the thread kernel (one env per 2^shift lanes).  Measured: it does NOT
// pay, because the kernel is bound by its local-memory traffic (6.5 KB of spilled constraint
// rows per env): with idle lanes in between, every spilled word still moves a full
// 32-byte sector.  Default 0; ENVPOOL_B200_HC_LANE_SHIFT (0..5) keeps the experiment runnable.
static int hc_lane_shift(int) {
  static const int forced = [] {
    const char* e = getenv("ENVPOOL_B200_HC_LANE_SHIFT");
    return e ? atoi(e) : -1;
  }();
  return (forced >= 0 && forced <= 5) ? forced : 0;
}

// Rows per lane kept in shared memory: everything (27) while one CTA per SM covers the batch,
// less as more CTAs share an SM (at most 4: what the kernel's registers allow).
// ENVPOOL_B200_HC_PAIR_KS overrides (A/B switch).
static int pair_rows_in_smem(int n) {
  static const int forced = [] {
    const char* e = getenv("ENVPOOL_B200_HC_PAIR_KS");
    return e ? atoi(e) : 0;
  }();
  if (forced >= kPairKsMin && forced <= hcp::MAXR) return forced;
  const int sms = device_sm_count();
  const int ctas = (2 * n + kPairBlock - 1) / kPairBlock;
  int per_sm = (ctas + sms - 1) / sms;  // CTAs per SM for a single wave
  per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
  const int row_bytes = hcp::NF * kPairBlock * (int)sizeof(double);
  int ks = (int)((216 * 1024 / per_sm) / row_bytes);
  ks = ks > hcp::MAXR ? hcp::MAXR : ks;
  return ks < kPairKsMin ? kPairKsMin : ks;
}

int mjc_pair_rows(const MjcPool* m, int n) { return m->variant == 0 ? pair_rows_in_smem(n) : 0; }

static void launch_pair(MjcPool* m, const StateView& sv, const OutView& ov, const double* d_action,
                        const int32_t* d_env_ids, int n, int force_reset, int T,
                        cudaStream_t stream) {
  // (Carrying fewer envs per warp -- every 2nd / 4th lane pair idle, so that a warp waits for
  // the slowest of 8 / 4 envs instead of 16 in the constraint solve -- was measured.  No gain; not
  // kept.)
  const int ks = pair_rows_in_smem(n);
  const int grid = (int)((2 * (int64_t)n + kPairBlock - 1) / kPairBlock);
  const size_t smem = (size_t)ks * hcp::NF * kPairBlock * sizeof(double);
  hc_pair_kernel<<<grid, kPairBlock, smem, stream>>>(sv, ov, m->prm, d_action, d_env_ids, n,
                                                     force_reset, T, ks);
}

cudaError_t mjc_launch_step(MjcPool* m, const StateView& sv, const OutView& ov,
                            const double* d_action, const int32_t* d_env_ids, int n,
                            int force_reset, cudaStream_t stream) {
  if (m->variant == 0) {
    launch_pair(m, sv, ov, d_action, d_env_ids, n, force_reset, 1, stream);
  } else if (m->variant == 2) {
    int grid = (n + kWarps - 1) / kWarps;
    hc_kernel<<<grid, kWarps * 32, 0, stream>>>(sv, ov, m->prm, d_action, d_env_ids, n,
                                                force_reset, 1);
  } else {
    const int sh = hc_lane_shift(n);
    int grid = (int)((((int64_t)n << sh) + kThreadBlock - 1) / kThreadBlock);
    hc_thread_kernel<<<grid, kThreadBlock, 0, stream>>>(sv, ov, m->prm, d_action, d_env_ids,
                                                        n, force_reset, 1, sh);
  }
  return cudaGetLastError();
}
cudaError_t mjc_launch_rollout(MjcPool* m, const StateView& sv, const OutView& ov,
                               const double* d_actions, int T, cudaStream_t stream) {
  int n = sv.n_envs;
  if (m->variant == 0) {
    launch_pair(m, sv, ov, d_actions, nullptr, n, 0, T, stream);
  } else if (m->variant == 2) {
    int grid = (n + kWarps - 1) / kWarps;
    hc_kernel<<<grid, kWarps * 32, 0, stream>>>(sv, ov, m->prm, d_actions, nullptr, n, 0, T);
  } else {
    const int sh = hc_lane_shift(n);
    int grid = (int)((((int64_t)n << sh) + kThreadBlock - 1) / kThreadBlock);
    hc_thread_kernel<<<grid, kThreadBlock, 0, stream>>>(sv, ov, m->prm, d_actions, nullptr, n,
                                                        0, T, sh);
  }
  return cudaGetLastError();
}

}  // namespace epb
