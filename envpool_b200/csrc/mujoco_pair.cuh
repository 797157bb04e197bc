// HalfCheetah physics, TWO LANES PER ENV.
//
// The cheetah's kinematic tree is torso | back leg | front leg, and every matrix of the
// step -- M, H = M + J^T D J, M + h B -- is block-arrow over exactly that split (no
// constraint row touches both legs).  Lane `side` (0 = back, 1 = front) of a lane pair owns
// ONE leg: its three hinges, three bodies, three capsules, its joint limits and contacts,
// its diagonal block A and its coupling block C.  The 3-dof root block is DUPLICATED: both
// lanes hold the same root state and run the same root arithmetic on bit-identical inputs,
// so both take the same branches (solver termination, line search) without ever exchanging a
// decision.  What a lane cannot know -- its partner's contribution to a root quantity -- is a
// `psum`: own + __shfl_xor(own, 1).  IEEE addition is commutative, so both lanes get the same
// bits; every root value is formed as  local_part + psum(leg_part)  in that order.
//
// Both lanes execute the SAME instruction stream (SIMT-friendly: no role divergence), each on
// half the rows, half of the kinematic chain and 21 instead of 36 matrix entries; a warp
// carries 16 envs.  Against one thread per env, the dependent chain of one mj_step is ~0.6x
// as long, nothing is indexed by a runtime leg id (which put H, fc and the solver vectors
// into local memory there), and the constraint rows of a lane live in shared memory (first
// `ks` rows; the rare rest in thread-local overflow).
//
// Dual build: with HCP_HOST defined this header compiles as plain C++ (two host threads play
// the lane pair and meet at every exchange, tests/hc_pair_host/); the CPU test suite checks
// that build against the independent CPU restatement of the same pipeline, so the pair algorithm
// is verified without a GPU.
#pragma once

#include "mujoco_model.h"

#if defined(HCP_HOST)
#include <cmath>
#define HCP_FN static inline
#define HCP_MFN inline
#define HCP_NOINLINE static
namespace epb {
namespace hcp {
double host_xch(void* chan, int side, double v);  // provided by the host harness
inline double hcp_rsqrt(double x) { return 1.0 / std::sqrt(x); }
inline void hcp_sincos(double x, double* s, double* c) { *s = std::sin(x); *c = std::cos(x); }
}  // namespace hcp
}  // namespace epb
#else
#define HCP_FN __device__ __forceinline__
#define HCP_MFN __device__ __forceinline__
#define HCP_NOINLINE __device__ __noinline__
namespace epb {
namespace hcp {
__device__ __forceinline__ double hcp_rsqrt(double x) { return rsqrt(x); }
__device__ __noinline__ void hcp_sincos(double x, double* s, double* c) { sincos(x, s, c); }
}  // namespace hcp
}  // namespace epb
#endif

namespace epb {
namespace hcp {

using hcm::HcModel;
using hcm::LegModel;
using hcm::MINVAL;
using hcm::MINIMP;
using hcm::MAXIMP;

constexpr int MAXR = 3 + 3 * 8;  // per lane: 3 joint limits + 8 contact sites x 3 merged rows
constexpr int NF = 10;           // doubles per row: jr[3] jl[3] D aref jar Jv
enum { F_JR = 0, F_JL = 3, F_D = 6, F_AREF = 7, F_JAR = 8, F_JV = 9 };

// What a lane needs besides its registers.
struct Ctx {
  int side;       // 0 = back leg + torso capsule, 1 = front leg + head capsule
  unsigned pm;    // device: the two-lane mask of this pair
  void* chan;     // host build: the rendezvous of the two threads
  double* srow;   // shared-memory rows of this lane: field f of row r at
                  // srow[(r*NF+f)*HCP_SSTRIDE], HCP_SSTRIDE = threads per CTA (rows are
                  // interleaved by thread: conflict-free)
  int ks;         // rows held in shared memory; rows >= ks go to ovf
  double* ovf;    // [MAXR - ks][NF] thread-local overflow
};

HCP_FN double xch(const Ctx& c, double v) {
#if defined(HCP_HOST)
  return host_xch(c.chan, c.side, v);
#else
  return __shfl_xor_sync(c.pm, v, 1);
#endif
}
// own + partner's: bit-identical on both lanes
HCP_FN double psum(const Ctx& c, double v) { return v + xch(c, v); }

// Solver branch trace of the host test build (HCP_STATS; tests/hc_pair_host/pair_stats.cc
// provides hcp_trace).  Each lane reports every branch its solver takes, as (event, value):
#if defined(HCP_STATS)
enum {
  TR_ROWS = 1,  // start of a constraint solve; value: rows of both lanes (0 = free flight)
  TR_WARM,      // warm start; value: 1 if qacc_smooth was taken, + 2 if cw == cs
  TR_LS,        // a Newton step's line search; value: TR_RUN, TR_SKIP_GS (!(gs < 0)), TR_SKIP_TOL
  TR_UPD,       // a line-search update of alpha; value: TR_NEWTON, TR_EXPAND, TR_BISECT
  TR_LS_END,    // how a line search that ran ended; value: TR_CONV, TR_STALL, TR_CAP
  TR_EXIT,      // how the Newton loop ended; value: TR_GRAD0, TR_COST, TR_GRAD, TR_MAXITER, TR_ALPHA0
};
enum { TR_RUN = 0, TR_SKIP_GS, TR_SKIP_TOL };
enum { TR_NEWTON = 0, TR_EXPAND, TR_BISECT };
enum { TR_CONV = 0, TR_STALL, TR_CAP };
enum { TR_GRAD0 = 0, TR_COST, TR_GRAD, TR_MAXITER, TR_ALPHA0 };
#define HCP_TRACE(c, ev, val) hcp_trace((c).side, (ev), (val))
// ... and the qacc_smooth it computed (root part, own leg part)
#define HCP_TRACE_SMOOTH(c, r, l) hcp_trace_smooth((c).side, (r), (l))
#else
#define HCP_TRACE_SMOOTH(c, r, l) ((void)0)
#define HCP_TRACE(c, ev, val) ((void)0)
#endif

// Row r of this lane: in shared memory (r < ks; field f at p[f * stride], stride = threads per
// CTA, a compile-time constant on the device so every access is an LDS with an immediate
// offset) or in the thread-local overflow (contiguous).  `with_row` runs `body` on whichever it
// is; the body is instantiated once per storage class.
#if defined(HCP_HOST)
#define HCP_SSTRIDE 1
#else
#define HCP_SSTRIDE 64
#endif
struct RowS {
  double* p;
  HCP_MFN double& operator[](int f) const { return p[f * HCP_SSTRIDE]; }
};
struct RowO {
  double* p;
  HCP_MFN double& operator[](int f) const { return p[f]; }
};
template <class F>
HCP_FN void with_row(const Ctx& c, int r, F&& body) {
  if (r < c.ks) {
    body(RowS{c.srow + r * (NF * HCP_SSTRIDE)});
  } else {
    body(RowO{c.ovf + (r - c.ks) * NF});
  }
}
// body(row) for rows 0..n-1 in order: the shared-memory rows, then the (rare) overflow rows
template <class F>
HCP_FN void for_rows(const Ctx& c, int n, F&& body) {
  const int ns = n < c.ks ? n : c.ks;
  for (int r = 0; r < ns; ++r) body(RowS{c.srow + r * (NF * HCP_SSTRIDE)});
  for (int r = c.ks; r < n; ++r) body(RowO{c.ovf + (r - c.ks) * NF});
}

// ---- packed symmetric 3x3: [0]=(0,0) [1]=(1,0) [2]=(1,1) [3]=(2,0) [4]=(2,1) [5]=(2,2) -------
HCP_FN void symv3(const double* A, const double* x, double* y) {
  y[0] = A[0] * x[0] + A[1] * x[1] + A[3] * x[2];
  y[1] = A[1] * x[0] + A[2] * x[1] + A[4] * x[2];
  y[2] = A[3] * x[0] + A[4] * x[1] + A[5] * x[2];
}
// in-place Cholesky A = L L^T; the diagonal of L is stored INVERTED
HCP_FN void chol3(double* A) {
  double d0 = hcp_rsqrt(A[0]);
  double l10 = A[1] * d0, l20 = A[3] * d0;
  double d1 = hcp_rsqrt(A[2] - l10 * l10);
  double l21 = (A[4] - l20 * l10) * d1;
  double d2 = hcp_rsqrt(A[5] - l20 * l20 - l21 * l21);
  A[0] = d0; A[1] = l10; A[2] = d1; A[3] = l20; A[4] = l21; A[5] = d2;
}
HCP_FN void fwd3(const double* L, double* x) {  // x <- L^-1 x
  x[0] = x[0] * L[0];
  x[1] = (x[1] - L[1] * x[0]) * L[2];
  x[2] = (x[2] - L[3] * x[0] - L[4] * x[1]) * L[5];
}
HCP_FN void bwd3(const double* L, double* x) {  // x <- L^-T x
  x[2] = x[2] * L[5];
  x[1] = (x[1] - L[4] * x[2]) * L[2];
  x[0] = (x[0] - L[1] * x[1] - L[3] * x[2]) * L[0];
}

// Block-arrow matrix as one lane holds it: root block R (duplicated), own leg block A, own
// coupling C[leg dof][root dof].
struct Arrow {
  double R[6], A[6], C[3][3];
};
// Its factorisation, leaves first (what MuJoCo's sparse L^T D L does on the kinematic tree):
//   A = LA LA^T,  W = LA^-1 C,  S = R - W_b^T W_b - W_f^T W_f = LS LS^T
struct Fac {
  double LA[6], W[3][3], LS[6];
};

HCP_FN void pair_factor(const Ctx& c, const Arrow& H, Fac& f) {
#pragma unroll
  for (int t = 0; t < 6; ++t) f.LA[t] = H.A[t];
  chol3(f.LA);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double col[3] = {H.C[0][r], H.C[1][r], H.C[2][r]};
    fwd3(f.LA, col);
    f.W[0][r] = col[0]; f.W[1][r] = col[1]; f.W[2][r] = col[2];
  }
  double own[6];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j)
      own[i * (i + 1) / 2 + j] =
          f.W[0][i] * f.W[0][j] + f.W[1][i] * f.W[1][j] + f.W[2][i] * f.W[2][j];
#pragma unroll
  for (int t = 0; t < 6; ++t) f.LS[t] = H.R[t] - psum(c, own[t]);
  chol3(f.LS);
}
// solve H x = g in place: gr root part (duplicated), gl own leg part
HCP_FN void pair_apply(const Ctx& c, const Fac& f, double* gr, double* gl) {
  fwd3(f.LA, gl);
  double t[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) t[r] = f.W[0][r] * gl[0] + f.W[1][r] * gl[1] + f.W[2][r] * gl[2];
#pragma unroll
  for (int r = 0; r < 3; ++r) gr[r] -= psum(c, t[r]);
  fwd3(f.LS, gr);
  bwd3(f.LS, gr);
#pragma unroll
  for (int l = 0; l < 3; ++l) gl[l] -= f.W[l][0] * gr[0] + f.W[l][1] * gr[1] + f.W[l][2] * gr[2];
  bwd3(f.LA, gl);
}
// y = H x
HCP_FN void pair_mv(const Ctx& c, const Arrow& H, const double* xr, const double* xl, double* yr,
                    double* yl) {
  symv3(H.R, xr, yr);
  symv3(H.A, xl, yl);
  double t[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) t[r] = H.C[0][r] * xl[0] + H.C[1][r] * xl[1] + H.C[2][r] * xl[2];
#pragma unroll
  for (int r = 0; r < 3; ++r) yr[r] += psum(c, t[r]);
#pragma unroll
  for (int l = 0; l < 3; ++l) yl[l] += H.C[l][0] * xr[0] + H.C[l][1] * xr[1] + H.C[l][2] * xr[2];
}

template <class Row>
HCP_FN double row_dot(const Row& q, const double* xr, const double* xl) {
  return q[F_JR + 0] * xr[0] + q[F_JR + 1] * xr[1] + q[F_JR + 2] * xr[2] +
         q[F_JL + 0] * xl[0] + q[F_JL + 1] * xl[1] + q[F_JL + 2] * xl[2];
}

// mj_makeImpedance for one constraint class k (0 = contact, 1 = joint limit): the impedance at
// penetration `pos` (solimp midpoint 0.5, power 2: MuJoCo's defaults for the entries the XML
// leaves out).  Everything that does not depend on `pos` -- the clamped dmin / dmax, 1 / width,
// and the spring-damper K, B of solref -- is precomputed in the model (fill_impedance_constants).
HCP_FN double pair_imp(const HcModel& cm, int k, double pos) {
  const double dmin = cm.imp_dmin[k], dmax = cm.imp_dmax[k];
  const double x = fabs(pos) * cm.imp_invwidth[k];
  const double u = 1 - x;
  const double y = x <= 0.5 ? 2 * (x * x) : 1 - 2 * (u * u);
  const double imp = dmin + y * (dmax - dmin);
  return x >= 1 ? dmax : (x <= 0 ? dmin : imp);
}

// Per-lane state: the root part is the same in both lanes of a pair.
struct PairState {
  double qr[3], vr[3], wr[3];  // rootx, rootz, rooty: qpos, qvel, qacc_warmstart
  double ql[3], vl[3], wl[3];  // own leg: thigh, shin, foot hinges
  double ctrl[3];              // own leg's actuators
};

// One mj_step of one env, executed by its lane pair.  `cm` is the model (constant memory on
// the device), `L` this lane's leg table.
HCP_FN void pair_substep(const Ctx& c, const HcModel& cm, const LegModel& L, PairState& s) {
  // ---- kinematics: torso (duplicated) and own leg, thigh -> shin -> foot -------------------
  double c0, sn0, cb[3], sb[3], om[3];
  {
    double th0 = s.qr[2], th[3];
    th[0] = th0 + s.ql[0]; th[1] = th[0] + s.ql[1]; th[2] = th[1] + s.ql[2];
    om[0] = s.vr[2] + s.vl[0]; om[1] = om[0] + s.vl[1]; om[2] = om[1] + s.vl[2];
    hcp_sincos(th0, &sn0, &c0);
#pragma unroll
    for (int k = 0; k < 3; ++k) hcp_sincos(th[k], &sb[k], &cb[k]);
  }
  const double om0 = s.vr[2];
  const double ox0 = cm.bposx[0] + s.qr[0], oz0 = cm.bposz[0] + s.qr[1];
  double ox[3], oz[3], aox[3], aoz[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double cp = k ? cb[k - 1] : c0, sp = k ? sb[k - 1] : sn0, omp = k ? om[k - 1] : om0;
    const double rx = cp * L.bposx[k] + sp * L.bposz[k];
    const double rz = -sp * L.bposx[k] + cp * L.bposz[k];
    ox[k] = (k ? ox[k - 1] : ox0) + rx;
    oz[k] = (k ? oz[k - 1] : oz0) + rz;
    const double op2 = omp * omp;
    aox[k] = (k ? aox[k - 1] : 0.0) - op2 * rx;
    aoz[k] = (k ? aoz[k - 1] : 0.0) - op2 * rz;
  }
  // CoM, inertial force m (a - g) and its moment about the world origin, per body
  double cx0, cz0, fx0, fz0, tq0;
  {
    const double rx = c0 * cm.comx[0] + sn0 * cm.comz[0];
    const double rz = -sn0 * cm.comx[0] + c0 * cm.comz[0];
    cx0 = ox0 + rx;
    cz0 = oz0 + rz;
    const double o2 = om0 * om0;
    fx0 = cm.mass[0] * (0.0 - o2 * rx);
    fz0 = cm.mass[0] * (0.0 - o2 * rz - cm.gravity);
    tq0 = cz0 * fx0 - cx0 * fz0;
  }
  double Cm[3], Ccx[3], Ccz[3], Ci[3], fx[3], fz[3], tq[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double rx = cb[k] * L.comx[k] + sb[k] * L.comz[k];
    const double rz = -sb[k] * L.comx[k] + cb[k] * L.comz[k];
    Ccx[k] = ox[k] + rx;
    Ccz[k] = oz[k] + rz;
    Cm[k] = L.mass[k];
    Ci[k] = L.iyy[k];
    const double o2 = om[k] * om[k];
    fx[k] = L.mass[k] * (aox[k] - o2 * rx);
    fz[k] = L.mass[k] * (aoz[k] - o2 * rz - cm.gravity);
    tq[k] = Ccz[k] * fx[k] - Ccx[k] * fz[k];
  }
  // ---- composite bodies of the leg, foot -> shin -> thigh (mj_crb), force sums (mj_rne) ------
#pragma unroll
  for (int child = 2; child >= 1; --child) {
    const int par = child - 1;
    const double m = Cm[par] + Cm[child];
    const double minv = 1.0 / m;
    const double nx = (Cm[par] * Ccx[par] + Cm[child] * Ccx[child]) * minv;
    const double nz = (Cm[par] * Ccz[par] + Cm[child] * Ccz[child]) * minv;
    const double dpx = Ccx[par] - nx, dpz = Ccz[par] - nz;
    const double dcx = Ccx[child] - nx, dcz = Ccz[child] - nz;
    Ci[par] = Ci[par] + Ci[child] + Cm[par] * (dpx * dpx + dpz * dpz) +
              Cm[child] * (dcx * dcx + dcz * dcz);
    Cm[par] = m; Ccx[par] = nx; Ccz[par] = nz;
    fx[par] += fx[child]; fz[par] += fz[child]; tq[par] += tq[child];
  }
  // ---- joint-space inertia (block arrow) + armature ------------------------------------------
  // Root block: the whole-tree composite about the torso origin = torso + psum(leg composite),
  // by the parallel-axis theorem term by term (no merge order to agree on).
  Arrow M;
  double fxs, fzs, tqs;  // subtree force sums at the root
  {
    const double dx = Ccx[0] - ox0, dz = Ccz[0] - oz0;
    const double lm = psum(c, Cm[0]);
    const double lmz = psum(c, Cm[0] * dz);
    const double lmx = psum(c, Cm[0] * dx);
    const double li = psum(c, Ci[0] + Cm[0] * (dx * dx + dz * dz));
    const double tx = cx0 - ox0, tz = cz0 - oz0;
    const double mt = cm.mass[0] + lm;
    M.R[0] = mt; M.R[1] = 0; M.R[2] = mt;
    M.R[3] = cm.mass[0] * tz + lmz;
    M.R[4] = -(cm.mass[0] * tx + lmx);
    M.R[5] = cm.iyy[0] + cm.mass[0] * (tx * tx + tz * tz) + li + cm.armature[2];
    fxs = fx0 + psum(c, fx[0]);
    fzs = fz0 + psum(c, fz[0]);
    tqs = tq0 + psum(c, tq[0]);
  }
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    const double rx = Ccx[l] - ox[l], rz = Ccz[l] - oz[l];
    M.C[l][0] = Cm[l] * rz;
    M.C[l][1] = -Cm[l] * rx;
    M.C[l][2] = Ci[l] + Cm[l] * (rx * (Ccx[l] - ox0) + rz * (Ccz[l] - oz0));
#pragma unroll
    for (int j = 0; j <= l; ++j) {
      double v = Ci[l] + Cm[l] * (rx * (Ccx[l] - ox[j]) + rz * (Ccz[l] - oz[j]));
      if (j == l) v += L.armature[l];
      M.A[l * (l + 1) / 2 + j] = v;
    }
  }
  // ---- bias, passive, actuation -> qfrc_smooth; qacc_smooth ----------------------------------
  double fsr[3], fsl[3];
  fsr[0] = -fxs;
  fsr[1] = -fzs;
  fsr[2] = -(tqs - oz0 * fxs + ox0 * fzs);
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    const double bias = tq[l] - oz[l] * fx[l] + ox[l] * fz[l];
    double u = s.ctrl[l];
    u = u < -1 ? -1 : (u > 1 ? 1 : u);
    fsl[l] = -L.stiffness[l] * s.ql[l] - L.damping[l] * s.vl[l] - bias + L.gear[l] * u;
  }
  Fac FM;
  pair_factor(c, M, FM);
  double asr[3], asl[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) { asr[i] = fsr[i]; asl[i] = fsl[i]; }
  pair_apply(c, FM, asr, asl);
  HCP_TRACE_SMOOTH(c, asr, asl);
  // ---- collision + constraint rows of this lane ------------------------------------------------
  int n = 0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {  // joint limits (mj_instantiateLimit)
    const double dlo = s.ql[j] - L.rlo[j], dhi = L.rhi[j] - s.ql[j];
    const bool lo = dlo < 0, hi = !lo && dhi < 0;
    if (lo || hi) {
      const double sign = lo ? 1.0 : -1.0, dist = lo ? dlo : dhi;
      const double imp = pair_imp(cm, 1, dist);
      // D = 1 / R, R = max(MINVAL, (1 - imp) * diagApprox / imp): one division
      const double D = imp / fmax(MINVAL * imp, (1 - imp) * L.dof_invw[j]);
      const double aref = -cm.imp_B[1] * (sign * s.vl[j]) - cm.imp_K[1] * imp * dist;
      with_row(c, n++, [&](auto q) {
        q[F_JR + 0] = 0; q[F_JR + 1] = 0; q[F_JR + 2] = 0;
        q[F_JL + 0] = j == 0 ? sign : 0.0;
        q[F_JL + 1] = j == 1 ? sign : 0.0;
        q[F_JL + 2] = j == 2 ? sign : 0.0;
        q[F_D] = D;
        q[F_AREF] = aref;
      });
    }
  }
#pragma unroll 1
  for (int g = 0; g < 4; ++g) {  // floor plane vs the end spheres of this lane's capsules
    const int lvl = g - 1;       // -1: a capsule of the torso body
    const double cg = g == 0 ? c0 : (g == 1 ? cb[0] : (g == 2 ? cb[1] : cb[2]));
    const double sg_ = g == 0 ? sn0 : (g == 1 ? sb[0] : (g == 2 ? sb[1] : sb[2]));
    const double bx = g == 0 ? ox0 : (g == 1 ? ox[0] : (g == 2 ? ox[1] : ox[2]));
    const double bz = g == 0 ? oz0 : (g == 1 ? oz[0] : (g == 2 ? oz[1] : oz[2]));
    const double gx = bx + cg * L.gposx[g] + sg_ * L.gposz[g];
    const double gz = bz - sg_ * L.gposx[g] + cg * L.gposz[g];
    const double ax = cg * L.gaxx[g] + sg_ * L.gaxz[g];
    const double az = -sg_ * L.gaxx[g] + cg * L.gaxz[g];
#pragma unroll 1
    for (int en = 0; en < 2; ++en) {
      const double sg = en ? -1.0 : 1.0;
      const double pz = gz + sg * L.ghalf[g] * az;
      if (pz > cm.grad) continue;
      const double px = gx + sg * L.ghalf[g] * ax;
      const double dist = pz - cm.grad;
      const double cpz = pz - (cm.grad + dist / 2);  // sphere centre - n (radius + dist/2)
      // point Jacobian: root dofs, then this leg's hinges down to the body's level
      const double jx2 = cpz - oz0, jz2 = -(px - ox0);
      double lx[3], lz[3];
#pragma unroll
      for (int l = 0; l < 3; ++l) {
        lx[l] = (l <= lvl) ? cpz - oz[l] : 0.0;
        lz[l] = (l <= lvl) ? -(px - ox[l]) : 0.0;
      }
      const double velx = s.vr[0] + jx2 * s.vr[2] + lx[0] * s.vl[0] + lx[1] * s.vl[1] + lx[2] * s.vl[2];
      const double velz = s.vr[1] + jz2 * s.vr[2] + lz[0] * s.vl[0] + lz[1] * s.vl[1] + lz[2] * s.vl[2];
      const double imp = pair_imp(cm, 0, dist);
      const double tran = L.invw_tran[g];
      const double dA = tran + cm.mu * cm.mu * tran;
      // D = 1 / R, R = max(MINVAL, (1 - imp) * dA / imp) * 2 mu^2: one division
      const double D = imp / (fmax(MINVAL * imp, (1 - imp) * dA) * (2 * cm.mu * cm.mu));
      const double B = cm.imp_B[0], kip = cm.imp_K[0] * imp * dist;
      // pyramid edges n + mu t, n - mu t; the two edges along +-y coincide with n in the
      // plane and are merged into one row of weight 2 D
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const double sm = e == 0 ? cm.mu : (e == 1 ? -cm.mu : 0.0);
        with_row(c, n + e, [&](auto q) {
          q[F_JR + 0] = sm;   // jz[0] + sm * jx[0] = 0 + sm * 1
          q[F_JR + 1] = 1.0;  // jz[1] + sm * jx[1] = 1 + sm * 0
          q[F_JR + 2] = jz2 + sm * jx2;
          q[F_JL + 0] = lz[0] + sm * lx[0];
          q[F_JL + 1] = lz[1] + sm * lx[1];
          q[F_JL + 2] = lz[2] + sm * lx[2];
          q[F_D] = e == 2 ? 2 * D : D;
          q[F_AREF] = -B * (velz + sm * velx) - kip;
        });
      }
      n += 3;
    }
  }
  // ---- constraint solve (Newton, exact line search), pair-cooperative ------------------------
  double ar[3], al[3], fcr[3], fcl[3];
  const double ntot = psum(c, (double)n);
  HCP_TRACE(c, TR_ROWS, (int)ntot);
  if (ntot == 0) {
#pragma unroll
    for (int i = 0; i < 3; ++i) { ar[i] = asr[i]; al[i] = asl[i]; fcr[i] = 0; fcl[i] = 0; }
  } else {
    double Mar[3], Mal[3], gr[3], gl[3], sr[3], sl[3], Mvr[3], Mvl[3];
    {  // warmstart: the better of qacc_warmstart and qacc_smooth
      double cw = 0, cs = 0;
      for_rows(c, n, [&](auto q) {
        const double aref = q[F_AREF], D = q[F_D];
        const double sw = row_dot(q, s.wr, s.wl) - aref;
        const double ss = row_dot(q, asr, asl) - aref;
        if (sw < 0) cw += 0.5 * D * sw * sw;
        if (ss < 0) cs += 0.5 * D * ss * ss;
      });
      pair_mv(c, M, s.wr, s.wl, Mar, Mal);
#pragma unroll
      for (int i = 0; i < 3; ++i) cw += 0.5 * (Mal[i] - fsl[i]) * (s.wl[i] - asl[i]);
      double gw = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) gw += 0.5 * (Mar[i] - fsr[i]) * (s.wr[i] - asr[i]);
      cw = gw + psum(c, cw);
      cs = psum(c, cs);
      const bool use_smooth = cw > cs;
      HCP_TRACE(c, TR_WARM, (use_smooth ? 1 : 0) + (cw == cs ? 2 : 0));
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        ar[i] = use_smooth ? asr[i] : s.wr[i];
        al[i] = use_smooth ? asl[i] : s.wl[i];
      }
    }
    const double scale = 1.0 / (cm.meaninertia * hcm::NV);
    double cost = 0;
    for (int iter = 0; iter <= cm.max_iter; ++iter) {
      pair_mv(c, M, ar, al, Mar, Mal);
      Arrow H = M;
      double fo[3] = {0, 0, 0}, ho[6] = {0, 0, 0, 0, 0, 0}, co = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) fcl[i] = 0;
      for_rows(c, n, [&](auto q) {
        const double j0 = q[F_JR + 0], j1 = q[F_JR + 1], j2 = q[F_JR + 2];
        const double l0 = q[F_JL + 0], l1 = q[F_JL + 1], l2 = q[F_JL + 2];
        const double D = q[F_D];
        const double sj = j0 * ar[0] + j1 * ar[1] + j2 * ar[2] + l0 * al[0] + l1 * al[1] +
                          l2 * al[2] - q[F_AREF];
        q[F_JAR] = sj;
        if (sj < 0) {
          const double f = -D * sj;
          co += 0.5 * D * sj * sj;
          fo[0] += j0 * f; fo[1] += j1 * f; fo[2] += j2 * f;
          ho[0] += D * j0 * j0; ho[1] += D * j1 * j0; ho[2] += D * j1 * j1;
          ho[3] += D * j2 * j0; ho[4] += D * j2 * j1; ho[5] += D * j2 * j2;
          fcl[0] += l0 * f; fcl[1] += l1 * f; fcl[2] += l2 * f;
          H.A[0] += D * l0 * l0; H.A[1] += D * l1 * l0; H.A[2] += D * l1 * l1;
          H.A[3] += D * l2 * l0; H.A[4] += D * l2 * l1; H.A[5] += D * l2 * l2;
          H.C[0][0] += D * l0 * j0; H.C[0][1] += D * l0 * j1; H.C[0][2] += D * l0 * j2;
          H.C[1][0] += D * l1 * j0; H.C[1][1] += D * l1 * j1; H.C[1][2] += D * l1 * j2;
          H.C[2][0] += D * l2 * j0; H.C[2][1] += D * l2 * j1; H.C[2][2] += D * l2 * j2;
        }
      });
      double g2o = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        co += 0.5 * (Mal[i] - fsl[i]) * (al[i] - asl[i]);
        gl[i] = Mal[i] - fsl[i] - fcl[i];
        g2o += gl[i] * gl[i];
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) fcr[i] = psum(c, fo[i]);
#pragma unroll
      for (int t = 0; t < 6; ++t) H.R[t] += psum(c, ho[t]);
      double newcost = 0, g2 = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        newcost += 0.5 * (Mar[i] - fsr[i]) * (ar[i] - asr[i]);
        gr[i] = Mar[i] - fsr[i] - fcr[i];
        g2 += gr[i] * gr[i];
      }
      newcost += psum(c, co);
      g2 += psum(c, g2o);
      const double gnorm = sqrt(g2);
      if (iter > 0) {
        if (scale * (cost - newcost) < cm.tolerance || scale * gnorm < cm.tolerance) {
          HCP_TRACE(c, TR_EXIT, scale * (cost - newcost) < cm.tolerance ? TR_COST : TR_GRAD);
          break;
        }
      } else if (scale * gnorm < cm.tolerance) {
        HCP_TRACE(c, TR_EXIT, TR_GRAD0);
        break;
      }
      cost = newcost;
      if (iter == cm.max_iter) {
        HCP_TRACE(c, TR_EXIT, TR_MAXITER);
        break;
      }
      Fac FH;
      pair_factor(c, H, FH);
#pragma unroll
      for (int i = 0; i < 3; ++i) { sr[i] = gr[i]; sl[i] = gl[i]; }
      pair_apply(c, FH, sr, sl);
#pragma unroll
      for (int i = 0; i < 3; ++i) { sr[i] = -sr[i]; sl[i] = -sl[i]; }
      pair_mv(c, M, sr, sl, Mvr, Mvl);
      double q1 = 0, q2 = 0, sn2 = 0, gs = 0, q1o = 0, q2o = 0, sno = 0, gso = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        q1 += sr[i] * (Mar[i] - fsr[i]);
        q2 += sr[i] * Mvr[i];
        sn2 += sr[i] * sr[i];
        gs += sr[i] * gr[i];
        q1o += sl[i] * (Mal[i] - fsl[i]);
        q2o += sl[i] * Mvl[i];
        sno += sl[i] * sl[i];
        gso += sl[i] * gl[i];
      }
      q1 += psum(c, q1o);
      q2 += psum(c, q2o);
      sn2 += psum(c, sno);
      gs += psum(c, gso);
      // Exact line search on phi(alpha) = cost(a + alpha * search), by safeguarded Newton steps on
      // phi'; stop at |phi'(alpha)| < tolerance * ls_tolerance * |search| / scale (MuJoCo's scaled
      // gradient tolerance of the 1-D problem, ls_tolerance = 0.01).
      // The evaluation at alpha = 0 needs no pass over the rows: phi'(0) = grad . search, and
      // because search = -H^-1 grad with H built from exactly the rows active at alpha = 0,
      // phi''(0) = search . H search = -phi'(0): the first Newton step lands on alpha = 1.  So
      // the first row pass evaluates alpha = 1 -- fused with the pass that computes J search --
      // and in two of three line searches it is also the last (profiles/hc_pair_iteration_stats.py
      // prints the statistics of the host build).
      const double gtol = cm.tolerance * 0.01 * sqrt(sn2) / scale;
      double alpha = 0;
      HCP_TRACE(c, TR_LS, !(gs < 0) ? TR_SKIP_GS : (fabs(gs) < gtol ? TR_SKIP_TOL : TR_RUN));
      if (gs < 0 && !(fabs(gs) < gtol)) {
#if defined(HCP_STATS)
        int ls_end = TR_CAP;
#endif
        double lo = 0, hi = INFINITY;
        alpha = 1.0;
        double d1o = 0, d2o = 0;
        for_rows(c, n, [&](auto q) {
          const double jv = row_dot(q, sr, sl), D = q[F_D];
          q[F_JV] = jv;
          const double x = q[F_JAR] + jv;
          if (x < 0) {
            d1o += D * x * jv;
            d2o += D * jv * jv;
          }
        });
        for (int k = 1; k < cm.ls_iter; ++k) {
          if (k > 1) {
            d1o = 0;
            d2o = 0;
            for_rows(c, n, [&](auto q) {
              const double jv = q[F_JV], D = q[F_D];
              const double x = q[F_JAR] + alpha * jv;
              if (x < 0) {
                d1o += D * x * jv;
                d2o += D * jv * jv;
              }
            });
          }
          const double d1 = (q1 + alpha * q2) + psum(c, d1o);
          const double d2 = q2 + psum(c, d2o);
          if (fabs(d1) < gtol) {
#if defined(HCP_STATS)
            ls_end = TR_CONV;
#endif
            break;
          }
          if (d1 < 0) lo = alpha; else hi = alpha;
          double next = alpha - d1 / d2;
#if defined(HCP_STATS)
          const int upd = (next > lo && next < hi) ? TR_NEWTON : (hi == INFINITY ? TR_EXPAND : TR_BISECT);
#endif
          if (!(next > lo && next < hi)) next = (hi == INFINITY) ? 2 * alpha + 1 : 0.5 * (lo + hi);
          if (next == alpha) {
#if defined(HCP_STATS)
            ls_end = TR_STALL;
#endif
            break;
          }
          HCP_TRACE(c, TR_UPD, upd);
          alpha = next;
        }
        HCP_TRACE(c, TR_LS_END, ls_end);
      }
      if (alpha == 0) {
        HCP_TRACE(c, TR_EXIT, TR_ALPHA0);
        break;
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) { ar[i] += alpha * sr[i]; al[i] += alpha * sl[i]; }
    }
  }
  // ---- mj_Euler with implicit joint damping -------------------------------------------------------
  {
    Arrow E = M;
#pragma unroll
    for (int l = 0; l < 3; ++l) E.A[l * (l + 1) / 2 + l] += cm.timestep * L.damping[l];
    Fac FE;
    pair_factor(c, E, FE);
    double rr[3], rl[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { rr[i] = fsr[i] + fcr[i]; rl[i] = fsl[i] + fcl[i]; }
    pair_apply(c, FE, rr, rl);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double vr = s.vr[i] + cm.timestep * rr[i];
      s.vr[i] = vr;
      s.qr[i] += cm.timestep * vr;
      s.wr[i] = ar[i];
      const double vl = s.vl[i] + cm.timestep * rl[i];
      s.vl[i] = vl;
      s.ql[i] += cm.timestep * vl;
      s.wl[i] = al[i];
    }
  }
}

}  // namespace hcp
}  // namespace epb
