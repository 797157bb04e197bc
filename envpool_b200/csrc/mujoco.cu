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
// One kernel, hc_pair_kernel below: two lanes per env, one leg each (the physics of a lane is
// mujoco_pair.cuh).  Host side of the file: compile_half_cheetah (what mj_loadXML derives from
// the XML) and the launch plumbing.  Arithmetic is fp64 (the reference's); no dense
// contraction, no tensor cores.
//
// PARITY: unpinned against MuJoCo itself (MuJoCo is not a dependency of this project); pinned
// against the CPU restatement of the same pipeline (tests/ only).  See DESIGN.md section 3.
#include "mujoco.cuh"
#include "mujoco_model.h"
#include "mujoco_pair.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace epb {

namespace {

using hcm::NV; using hcm::NB; using hcm::NG; using hcm::NU;
using hcm::HcModel; using hcm::LegModel;
constexpr int kStateReals = 32;     // qpos[9] qvel[9] warm[9] norm_saved norm_has pad[3]

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

constexpr int kPairBlock = 64;  // threads per CTA = 32 envs
constexpr int kPairKsMin = 9;   // fewest constraint rows per lane ever held in shared memory
static_assert(kPairBlock == HCP_SSTRIDE, "row interleave stride = threads per CTA");

// the two LegModel tables in global memory (written at every pool creation, hc_setup): every
// CTA copies them into shared memory with one coalesced read
__device__ LegModel g_leg_model[2];

// One launch = T sync steps of `n` batch rows; TWO LANES PER ENV (mujoco_pair.cuh): lane
// 2*row is the back leg (and does everything that exists once per env: RNG, reward, the
// common columns), lane 2*row + 1 the front leg.  Dynamic shared memory: the first `ks`
// constraint rows of every lane, interleaved by thread.
//
// ptxas (CUDA 12.9, sm_90a): 255 registers, a 1904-byte stack frame (1440 B of it the
// thread-local row overflow `ovf`, (27 - 9) x 10 doubles), 340 B of spill stores and 556 B of
// spill loads: 4 CTAs (8 warps) per SM.  Builds capped at 144 and 128 registers (7 / 8 CTAs
// per SM: fewer waves) were measured and dropped: their spills cost more than the extra wave.
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

// On the pool's device (a second GPU needs its own copy of the symbols): the model, the leg
// tables and the kernel's shared-memory limit; the pool's HcParams from its configuration.
cudaError_t hc_setup(const epb_config& cfg, std::vector<char>& params) {
  static HcModel host_model;
  compile_half_cheetah(&host_model);
  cudaError_t e = cudaMemcpyToSymbol(cm, &host_model, sizeof(HcModel));
  LegModel legs[2];
  hcm::leg_model_of(host_model, 0, &legs[0]);
  hcm::leg_model_of(host_model, 1, &legs[1]);
  const int smem_max = hcp::MAXR * hcp::NF * kPairBlock * (int)sizeof(double);
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_leg_model, legs, sizeof(legs));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(hc_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             smem_max);
  HcParams prm;
  prm.frame_skip = cfg.frame_skip > 0 ? cfg.frame_skip : 5;
  // NaN = default (include/envpool_b200.h); any other value, negative included, as given
  prm.ctrl_cost_weight = std::isnan(cfg.ctrl_cost_weight) ? 0.1 : cfg.ctrl_cost_weight;
  prm.forward_reward_weight = std::isnan(cfg.forward_reward_weight) ? 1.0 : cfg.forward_reward_weight;
  prm.reset_noise_scale = std::isnan(cfg.reset_noise_scale) ? 0.1 : cfg.reset_noise_scale;
  params.resize(sizeof(prm));
  memcpy(params.data(), &prm, sizeof(prm));
  return e;
}

}  // namespace

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

int mjc_pair_rows(int n) { return pair_rows_in_smem(n); }

// T sync steps of n batch rows with the pool's HcParams (LaunchArgs::params)
static cudaError_t launch_pair(const LaunchArgs& a, const int32_t* env_ids, int n,
                               int force_reset, int T) {
  // (Carrying fewer envs per warp -- every 2nd / 4th lane pair idle, so that a warp waits for
  // the slowest of 8 / 4 envs instead of 16 in the constraint solve -- was measured.  No gain; not
  // kept.)
  const int ks = pair_rows_in_smem(n);
  const int grid = (int)((2 * (int64_t)n + kPairBlock - 1) / kPairBlock);
  const size_t smem = (size_t)ks * hcp::NF * kPairBlock * sizeof(double);
  hc_pair_kernel<<<grid, kPairBlock, smem, a.stream>>>(
      a.sv, a.ov, *static_cast<const HcParams*>(a.params), static_cast<const double*>(a.action),
      env_ids, n, force_reset, T, ks);
  return cudaGetLastError();
}
static cudaError_t hc_step(const LaunchArgs& a) {
  return launch_pair(a, a.env_ids, a.n, a.force_reset, 1);
}
static cudaError_t hc_rollout(const LaunchArgs& a) {
  return launch_pair(a, nullptr, a.sv.n_envs, 0, a.T);
}

// mujoco/gym/half_cheetah.h:44-62.  fp64 only (DESIGN.md); the step kernel has no peer-forwarding
// epilogue.  27 of the 32 state reals are live, so the dead 5 are taken off bytes_per_env_step.
const KindDesc kMujocoKinds[] = {{
    .kind = EPB_HALF_CHEETAH,
    .keys = {{"obs", EPB_F64, 1, {17}}, {"info:reward_run", EPB_F64, 0, {}},
             {"info:reward_ctrl", EPB_F64, 0, {}}, {"info:x_position", EPB_F64, 0, {}},
             {"info:x_velocity", EPB_F64, 0, {}}},
    .action = {"action", EPB_F64, 1, {NU}},
    .NR = kStateReals,
    .fp64_only = true,
    .launch = [](int, int) {
      return KindLaunch{hc_step, hc_rollout, nullptr, false, -2 * (kStateReals - 27) * 8};
    },
    .setup = hc_setup,
}};
const KindDesc* mujoco_kind(int kind) { return find_kind(kMujocoKinds, kind); }

}  // namespace epb
