// HalfCheetah model constants shared by the physics kernel (mujoco.cu, mujoco_pair.cuh) and
// by the host-side emulation of the pair-lane kernel used in the CPU tests.  Plain C++: no
// CUDA types.  What each field restates of
// third_party/mujoco_gym_xml_patches/half_cheetah_envpool.xml is documented where it is
// filled, compile_half_cheetah (mujoco.cu).
#pragma once

#if defined(__CUDACC__)
#define HCM_HD __host__ __device__
#else
#define HCM_HD
#endif

namespace epb {
namespace hcm {

constexpr int NV = 9, NB = 7, NG = 8, NU = 6;
constexpr double MINVAL = 1e-15, MINIMP = 0.0001, MAXIMP = 0.9999;

struct HcModel {
  double mass[NB], comx[NB], comz[NB], iyy[NB], bposx[NB], bposz[NB];
  double armature[NV], damping[NV], stiffness[NV], rlo[NV], rhi[NV];
  double gear[NU];
  double gposx[NG], gposz[NG], gaxx[NG], gaxz[NG], ghalf[NG];
  double dof_invweight0[NV], body_invw_tran[NB];
  double grad, timestep, gravity, mu, meaninertia, tolerance;
  double solref[2], solimp[3], solref_limit[2], solimp_limit[3];
  int parent[NB], depth[NB], gbody[NG];
  int chain_len[NB], chain[NB][4];  // hinge dofs from the root to the body, in order
  int chainmask[NB];                // bit d set iff hinge dof d is on the body's chain
  int max_iter, ls_iter;
  // what mj_makeImpedance needs per constraint class ([0] contact, [1] joint limit) that does
  // not depend on the penetration: clamped solimp dmin / dmax, 1 / width, and solref's
  // spring-damper  K = 1 / (dmax^2 tc^2 dr^2),  B = 2 / (dmax tc)
  double imp_dmin[2], imp_dmax[2], imp_invwidth[2], imp_K[2], imp_B[2];
};

inline void fill_impedance_constants(HcModel* m) {
  for (int k = 0; k < 2; ++k) {
    const double* solref = k ? m->solref_limit : m->solref;
    const double* solimp = k ? m->solimp_limit : m->solimp;
    const double lo = solimp[0] < MINIMP ? MINIMP : (solimp[0] > MAXIMP ? MAXIMP : solimp[0]);
    const double hi = solimp[1] < MINIMP ? MINIMP : (solimp[1] > MAXIMP ? MAXIMP : solimp[1]);
    m->imp_dmin[k] = lo;
    m->imp_dmax[k] = hi;
    m->imp_invwidth[k] = 1.0 / solimp[2];
    const double kd = hi * hi * solref[0] * solref[0] * solref[1] * solref[1];
    const double bd = hi * solref[0];
    m->imp_K[k] = 1.0 / (kd < MINVAL ? MINVAL : kd);
    m->imp_B[k] = 2.0 / (bd < MINVAL ? MINVAL : bd);
  }
}

// One leg of the cheetah as the pair-lane kernel sees it: side 0 = back leg (bodies 1-3,
// dofs 3-5, actuators 0-2, capsules 2-4) + the torso capsule (geom 0); side 1 = front leg
// (bodies 4-6, dofs 6-8, actuators 3-5, capsules 5-7) + the head capsule (geom 1).
struct LegModel {
  double mass[3], comx[3], comz[3], iyy[3], bposx[3], bposz[3];  // thigh, shin, foot
  double armature[3], damping[3], stiffness[3], rlo[3], rhi[3], gear[3], dof_invw[3];
  // geoms: slot 0 = this side's capsule of the TORSO body, slots 1..3 = the leg capsules
  double gposx[4], gposz[4], gaxx[4], gaxz[4], ghalf[4];
  double invw_tran[4];  // body_invweight0 (translation): torso, thigh, shin, foot
};

HCM_HD inline void leg_model_of(const HcModel& m, int side, LegModel* L) {
  for (int k = 0; k < 3; ++k) {
    const int b = 1 + 3 * side + k, i = 3 + 3 * side + k;
    L->mass[k] = m.mass[b]; L->comx[k] = m.comx[b]; L->comz[k] = m.comz[b];
    L->iyy[k] = m.iyy[b]; L->bposx[k] = m.bposx[b]; L->bposz[k] = m.bposz[b];
    L->armature[k] = m.armature[i]; L->damping[k] = m.damping[i];
    L->stiffness[k] = m.stiffness[i]; L->rlo[k] = m.rlo[i]; L->rhi[k] = m.rhi[i];
    L->gear[k] = m.gear[3 * side + k]; L->dof_invw[k] = m.dof_invweight0[i];
  }
  for (int s = 0; s < 4; ++s) {
    const int g = s == 0 ? side : 1 + 3 * side + s;
    L->gposx[s] = m.gposx[g]; L->gposz[s] = m.gposz[g];
    L->gaxx[s] = m.gaxx[g]; L->gaxz[s] = m.gaxz[g]; L->ghalf[s] = m.ghalf[g];
    L->invw_tran[s] = m.body_invw_tran[s == 0 ? 0 : 3 * side + s];
  }
}

}  // namespace hcm
}  // namespace epb
