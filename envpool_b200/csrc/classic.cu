// classic_control family: CartPole, Pendulum, Acrobot, MountainCar, MountainCarContinuous.
// One CUDA thread per env; state is R = double (reference arithmetic) or float (fast mode),
// outputs are the reference's float32 columns.  Each step() cites the reference lines it
// restates (paths relative to the reference tree's envpool/classic_control/).
//
// Compiled with -fmad=false: the reference is built for baseline x86-64 (no FMA), so the
// double path must not contract a*b+c either or trajectories drift from the reference.
#include <type_traits>

#include "common.cuh"

namespace epb {

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

__device__ __forceinline__ void sincos_small(double x, double* s, double* c);

template <typename R> struct M;
template <> struct M<double> {
  static __device__ __forceinline__ void sincos_small_(double x, double* s, double* c) {
    sincos_small(x, s, c);
  }
  static __device__ __forceinline__ double sin_(double x) { return sin(x); }
  static __device__ __forceinline__ double cos_(double x) { return cos(x); }
  // one argument reduction for both; same values as sin(x), cos(x)
  static __device__ __forceinline__ void sincos_(double x, double* s, double* c) { sincos(x, s, c); }
};
template <> struct M<float> {
  static __device__ __forceinline__ void sincos_small_(float x, float* s, float* c) {
    sincosf(x, s, c);
  }
  static __device__ __forceinline__ float sin_(float x) { return sinf(x); }
  static __device__ __forceinline__ float cos_(float x) { return cosf(x); }
  static __device__ __forceinline__ void sincos_(float x, float* s, float* c) { sincosf(x, s, c); }
};

// sin and cos of a SMALL angle (|x| <= 0.5 rad; CartPole's pole is inside +-0.21 while the
// episode lives): Taylor polynomials in x^2 to x^17 / x^16 (truncation < 2e-22, i.e. below
// half an ulp), two independent Horner chains of explicit FMAs -- no argument reduction, no
// quadrant selection, ~1/3 of the dependent latency of the generic routine.  Its results are
// within 1 ulp (0.62 ulp at most on an H100, tests/test_gpu_classic_model.py).  Larger angles
// take CUDA's sincos, which is within 2 ulp (1.42 ulp at most there on the envs' ranges).
__device__ __forceinline__ void sincos_small(double x, double* s, double* c) {
  if (fabs(x) > 0.5) {
    sincos(x, s, c);
    return;
  }
  const double z = __dmul_rn(x, x);
  double ps = -1.0 / 355687428096000.0;           // -1/17!
  ps = __fma_rn(ps, z, 1.0 / 1307674368000.0);    //  1/15!
  ps = __fma_rn(ps, z, -1.0 / 6227020800.0);      // -1/13!
  ps = __fma_rn(ps, z, 1.0 / 39916800.0);         //  1/11!
  ps = __fma_rn(ps, z, -1.0 / 362880.0);          // -1/9!
  ps = __fma_rn(ps, z, 1.0 / 5040.0);             //  1/7!
  ps = __fma_rn(ps, z, -1.0 / 120.0);             // -1/5!
  ps = __fma_rn(ps, z, 1.0 / 6.0);                //  1/3!  (sign folded below)
  double pc = 1.0 / 20922789888000.0;             //  1/16!
  pc = __fma_rn(pc, z, -1.0 / 87178291200.0);     // -1/14!
  pc = __fma_rn(pc, z, 1.0 / 479001600.0);        //  1/12!
  pc = __fma_rn(pc, z, -1.0 / 3628800.0);         // -1/10!
  pc = __fma_rn(pc, z, 1.0 / 40320.0);            //  1/8!
  pc = __fma_rn(pc, z, -1.0 / 720.0);             // -1/6!
  pc = __fma_rn(pc, z, 1.0 / 24.0);               //  1/4!
  pc = __fma_rn(pc, z, -0.5);                     // -1/2!
  // sin x = x - x^3 * (1/6 - z/120 + ...) ;  cos x = 1 + z * pc
  *s = __fma_rn(__dmul_rn(-x, z), ps, x);
  *c = __fma_rn(z, pc, 1.0);
}

template <typename R, int NR>
struct RealState {
  R v[NR];
};
template <typename R, int NR>
__device__ __forceinline__ void load_real(const StateView& sv, int eid, RealState<R, NR>& s) {
  const R* p = static_cast<const R*>(sv.rstate) + eid;
#pragma unroll
  for (int k = 0; k < NR; ++k) s.v[k] = p[(int64_t)k * sv.n_envs];
}
template <typename R, int NR>
__device__ __forceinline__ void store_real(const StateView& sv, int eid,
                                           const RealState<R, NR>& s) {
  R* p = static_cast<R*>(sv.rstate) + eid;
#pragma unroll
  for (int k = 0; k < NR; ++k) p[(int64_t)k * sv.n_envs] = s.v[k];
}

// Reset-ahead record of a RealState env: rec[e][slot] = NR reals, contiguous (8 / 16 / 32 B).
template <typename R, int NR>
__device__ __forceinline__ void load_rec_real(const StateView& sv, int eid, int slot,
                                              RealState<R, NR>& s) {
  constexpr int kBytes = NR * (int)sizeof(R);
  static_assert(kBytes == 8 || kBytes % 16 == 0, "record must be 8 bytes or 16-byte units");
  const char* p = static_cast<const char*>(sv.rec) +
                  ((int64_t)eid * sv.rec_q + slot) * kBytes;
  if constexpr (kBytes == 8) {
    uint2 q = *reinterpret_cast<const uint2*>(p);
    memcpy(&s.v[0], &q, 8);
  } else {
#pragma unroll
    for (int i = 0; i < kBytes / 16; ++i) {
      uint4 q = reinterpret_cast<const uint4*>(p)[i];
      memcpy(reinterpret_cast<char*>(&s.v[0]) + 16 * i, &q, 16);
    }
  }
}
template <typename R, int NR>
__device__ __forceinline__ void store_rec_real(const StateView& sv, int eid, int slot,
                                               const RealState<R, NR>& s) {
  constexpr int kBytes = NR * (int)sizeof(R);
  char* p = static_cast<char*>(sv.rec) + ((int64_t)eid * sv.rec_q + slot) * kBytes;
  if constexpr (kBytes == 8) {
    uint2 q;
    memcpy(&q, &s.v[0], 8);
    *reinterpret_cast<uint2*>(p) = q;
  } else {
#pragma unroll
    for (int i = 0; i < kBytes / 16; ++i) {
      uint4 q;
      memcpy(&q, reinterpret_cast<const char*>(&s.v[0]) + 16 * i, 16);
      reinterpret_cast<uint4*>(p)[i] = q;
    }
  }
}
template <typename R, int NR>
__device__ __forceinline__ void prefetch_rec_real(const StateView& sv, int eid, int slot) {
  constexpr int kBytes = NR * (int)sizeof(R);
  const char* p = static_cast<const char*>(sv.rec) +
                  ((int64_t)eid * sv.rec_q + slot) * kBytes;
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
#define EPB_REC_RESET_MEMBERS                                                               \
  static constexpr bool kRecReset = true;                                                   \
  static __device__ __forceinline__ void prefetch_rec(const StateView& sv, int e, int slot) { \
    prefetch_rec_real<typename std::remove_reference<decltype(State().v[0])>::type,         \
                      (int)(sizeof(State) / sizeof(State().v[0]))>(sv, e, slot);            \
  }                                                                                         \
  static __device__ __forceinline__ void load_rec(const StateView& sv, int e, int slot,     \
                                                  State& s) {                               \
    load_rec_real(sv, e, slot, s);                                                          \
  }                                                                                         \
  static __device__ __forceinline__ void store_rec(const StateView& sv, int e, int slot,    \
                                                   const State& s) {                        \
    store_rec_real(sv, e, slot, s);                                                         \
  }

// ----------------------------------------------------------------------------- CartPole
// cartpole.h:82-129
template <typename R>
struct CartPole {
  using Act = int32_t;
  using State = RealState<R, 4>;  // x, x_dot, theta, theta_dot
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = false;
  EPB_REC_RESET_MEMBERS
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    load_real(sv, e, s);
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    store_real(sv, e, s);
  }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    double v[4];
    rng->uniform_real_batch<4>(-0.05, 0.05, v);
#pragma unroll
    for (int k = 0; k < 4; ++k) s.v[k] = (R)v[k];
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt*, StepOut& so) {
    const R kGravity = (R)9.8, kMassPole = (R)0.1, kMassTotal = (R)(1.0 + 0.1);
    const R kLength = (R)0.5, kMassPoleLength = (R)(0.1 * 0.5), kForceMag = (R)10.0;
    const R kTau = (R)0.02, kThetaThresholdRadians = (R)(12 * 2 * M_PI / 360);
    const R kXThreshold = (R)2.4;
    R x = s.v[0], x_dot = s.v[1], theta = s.v[2], theta_dot = s.v[3];
    done = (cur >= sv.max_steps);
    R force = act == 1 ? kForceMag : -kForceMag;
    R costheta, sintheta;
    M<R>::sincos_small_(theta, &sintheta, &costheta);
    R temp = (force + kMassPoleLength * theta_dot * theta_dot * sintheta) / kMassTotal;
    R theta_acc = (kGravity * sintheta - costheta * temp) /
                  (kLength * ((R)(4.0 / 3.0) - kMassPole * costheta * costheta / kMassTotal));
    R x_acc = temp - kMassPoleLength * theta_acc * costheta / kMassTotal;
    x += kTau * x_dot;
    x_dot += kTau * x_acc;
    theta += kTau * theta_dot;
    theta_dot += kTau * theta_acc;
    if (x < -kXThreshold || x > kXThreshold || theta < -kThetaThresholdRadians ||
        theta > kThetaThresholdRadians) {
      done = 1;
    }
    s.v[0] = x; s.v[1] = x_dot; s.v[2] = theta; s.v[3] = theta_dot;
    so.reward = 1.0f;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (!ov.env[0]) return;
    float4 o = make_float4((float)s.v[0], (float)s.v[1], (float)s.v[2], (float)s.v[3]);
    static_cast<float4*>(ov.env[0])[row] = o;
  }
};

// ----------------------------------------------------------------------------- Pendulum
// pendulum.h:77-135
template <typename R>
struct Pendulum {
  using Act = float;
  using State = RealState<R, 2>;  // theta, theta_dot
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = false;
  EPB_REC_RESET_MEMBERS
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    load_real(sv, e, s);
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    store_real(sv, e, s);
  }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    uint32_t d[4];  // two uniform_real draws (different ranges), one round trip
    rng->next_batch<4>(d);
    s.v[0] = (R)__dadd_rn(__dmul_rn(Mt::canonical_from(d[0], d[1]), __dsub_rn(M_PI, -M_PI)),
                          -M_PI);
    s.v[1] = (R)__dadd_rn(__dmul_rn(Mt::canonical_from(d[2], d[3]), __dsub_rn(1.0, -1.0)),
                          -1.0);
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt*, StepOut& so) {
    const R kMaxSpeed = 8, kMaxTorque = 2, kDt = (R)0.05, kGravity = 10;
    const R kPi = (R)M_PI;
    R theta = s.v[0], theta_dot = s.v[1];
    done = (cur >= sv.max_steps);
    R u = act;
    if (act < -kMaxTorque) {
      u = -kMaxTorque;
    } else if (act > kMaxTorque) {
      u = kMaxTorque;
    }
    R cost = theta * theta + (R)0.1 * theta_dot * theta_dot + (R)0.001 * u * u;
    R new_theta_dot = theta_dot + 3 * (kGravity / 2 * M<R>::sin_(theta) + u) * kDt;
    // pendulum.h:104-113: both versions integrate theta with the UNCLIPPED new_theta_dot
    theta += new_theta_dot * kDt;
    theta_dot = new_theta_dot;
    if (new_theta_dot < -kMaxSpeed) {
      theta_dot = -kMaxSpeed;
    } else if (new_theta_dot > kMaxSpeed) {
      theta_dot = kMaxSpeed;
    }
    while (theta < -kPi) theta += kPi * 2;
    while (theta >= kPi) theta -= kPi * 2;
    s.v[0] = theta; s.v[1] = theta_dot;
    so.reward = (float)(-cost);
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (!ov.env[0]) return;
    float* o = static_cast<float*>(ov.env[0]) + row * 3;
    R sn, cs;
    M<R>::sincos_(s.v[0], &sn, &cs);
    o[0] = (float)cs;
    o[1] = (float)sn;
    o[2] = (float)s.v[1];
  }
};

// ------------------------------------------------------------------------------ Acrobot
// acrobot.h:94-191
template <typename R>
struct Acrobot {
  using Act = int32_t;
  using State = RealState<R, 4>;  // s0..s3 (s4 = torque is transient)
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = false;
  EPB_REC_RESET_MEMBERS
  struct V5 { R s0, s1, s2, s3, s4; };
  static __device__ __forceinline__ V5 add(V5 a, V5 b) {
    return V5{a.s0 + b.s0, a.s1 + b.s1, a.s2 + b.s2, a.s3 + b.s3, a.s4 + b.s4};
  }
  static __device__ __forceinline__ V5 mul(V5 a, R v) {
    return V5{a.s0 * v, a.s1 * v, a.s2 * v, a.s3 * v, a.s4 * v};
  }
  static __device__ __forceinline__ V5 derivs(V5 s) {  // acrobot.h:158-178
    const R kG = (R)9.8, kL = 1, kM = 1, kLC = (R)0.5, kI = 1;
    const R kHalfPi = (R)(M_PI / 2);
    R theta1 = s.s0, theta2 = s.s1, dtheta1 = s.s2, dtheta2 = s.s3, a = s.s4;
    R c2, s2;
    M<R>::sincos_(theta2, &s2, &c2);
    R d1 = kM * kLC * kLC + kM * (kL * kL + kLC * kLC + 2 * kL * kLC * c2) + kI * 2;
    R d2 = kM * (kLC * kLC + kL * kLC * c2) + kI;
    R phi2 = kM * kLC * kG * M<R>::cos_(theta1 + theta2 - kHalfPi);
    R phi1 = -(dtheta2 + 2 * dtheta1) * kM * kL * kLC * dtheta2 * s2 +
             kM * (kLC + kL) * kG * M<R>::cos_(theta1 - kHalfPi) + phi2;
    R ddtheta2 = (a + d2 / d1 * phi1 - kM * kL * kLC * dtheta1 * dtheta1 * s2 - phi2) /
                 (kM * kLC * kLC + kI - d2 * d2 / d1);
    R ddtheta1 = -(d2 * ddtheta2 + phi1) / d1;
    return V5{dtheta1, dtheta2, ddtheta1, ddtheta2, 0};
  }
  static __device__ __forceinline__ V5 rk4(V5 y0) {  // acrobot.h:150-156
    const R kDt = (R)0.2;
    V5 k1 = derivs(y0);
    V5 k2 = derivs(add(y0, mul(k1, kDt / 2)));
    V5 k3 = derivs(add(y0, mul(k2, kDt / 2)));
    V5 k4 = derivs(add(y0, mul(k3, kDt)));
    V5 sum = add(add(add(k1, mul(k2, 2)), mul(k3, 2)), k4);
    return add(y0, mul(sum, kDt / (R)6.0));
  }
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    load_real(sv, e, s);
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    store_real(sv, e, s);
  }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    double v[4];
    rng->uniform_real_batch<4>(-0.1, 0.1, v);
#pragma unroll
    for (int k = 0; k < 4; ++k) s.v[k] = (R)v[k];
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act act, int cur,
                                              int& done, Mt*, StepOut& so) {
    const R kPi = (R)M_PI, kMaxVel1 = (R)(4 * M_PI), kMaxVel2 = (R)(9 * M_PI);
    done = (cur >= sv.max_steps);
    float reward = -1.0f;
    V5 y = rk4(V5{s.v[0], s.v[1], s.v[2], s.v[3], (R)(act - 1)});
    while (y.s0 < -kPi) y.s0 += kPi * 2;
    while (y.s1 < -kPi) y.s1 += kPi * 2;
    while (y.s0 >= kPi) y.s0 -= kPi * 2;
    while (y.s1 >= kPi) y.s1 -= kPi * 2;
    if (y.s2 < -kMaxVel1) y.s2 = -kMaxVel1;
    if (y.s3 < -kMaxVel2) y.s3 = -kMaxVel2;
    if (y.s2 > kMaxVel1) y.s2 = kMaxVel1;
    if (y.s3 > kMaxVel2) y.s3 = kMaxVel2;
    if (-M<R>::cos_(y.s0) - M<R>::cos_(y.s0 + y.s1) > 1) {
      done = 1;
      reward = 0.0f;
    }
    s.v[0] = y.s0; s.v[1] = y.s1; s.v[2] = y.s2; s.v[3] = y.s3;
    so.reward = reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (ov.env[0]) {
      float2* o = reinterpret_cast<float2*>(static_cast<float*>(ov.env[0]) + row * 6);
      R s0, c0, s1, c1;
      M<R>::sincos_(s.v[0], &s0, &c0);
      M<R>::sincos_(s.v[1], &s1, &c1);
      o[0] = make_float2((float)c0, (float)s0);
      o[1] = make_float2((float)c1, (float)s1);
      o[2] = make_float2((float)s.v[2], (float)s.v[3]);
    }
    if (ov.env[1]) {
      static_cast<float2*>(ov.env[1])[row] = make_float2((float)s.v[0], (float)s.v[1]);
    }
  }
};

// ------------------------------------------------------------ MountainCar (+Continuous)
// mountain_car.h:76-119, mountain_car_continuous.h:77-127
template <typename R, bool kContinuous>
struct MountainCar {
  using Act = typename std::conditional<kContinuous, float, int32_t>::type;
  using State = RealState<R, 2>;  // pos, vel
  static constexpr bool kRngInReset = true, kRngInStep = false, kBlockObs = false;
  EPB_REC_RESET_MEMBERS
  static __device__ __forceinline__ void load(const StateView& sv, int e, State& s) {
    load_real(sv, e, s);
  }
  static __device__ __forceinline__ void store(const StateView& sv, int e, const State& s) {
    store_real(sv, e, s);
  }
  static __device__ __forceinline__ void reset(const StateView&, State& s, Mt* rng,
                                               StepOut& so) {
    s.v[0] = (R)rng->uniform_real(-0.6, -0.4);
    s.v[1] = 0;
    so.reward = 0.0f;
  }
  static __device__ __forceinline__ void step(const StateView& sv, State& s, Act action,
                                              int cur, int& done, Mt*, StepOut& so) {
    const R kMinPos = (R)-1.2, kMaxPos = (R)0.6, kMaxSpeed = (R)0.07;
    const R kGoalPos = kContinuous ? (R)0.45 : (R)0.5, kGoalVel = 0, kGravity = (R)0.0025;
    R pos = s.v[0], vel = s.v[1];
    done = (cur >= sv.max_steps);
    R act, reward;
    if (kContinuous) {
      act = (R)(float)action;
      reward = (R)-0.1 * act * act;
      if (act < -1) {
        act = -1;
      } else if (act > 1) {
        act = 1;
      }
      vel += act * (R)0.0015 - M<R>::cos_(3 * pos) * kGravity;
    } else {
      act = (R)((int)action - 1);
      reward = -1;
      vel += act * (R)0.001 - M<R>::cos_(3 * pos) * kGravity;
    }
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
    if (pos >= kGoalPos && vel >= kGoalVel) {
      done = 1;
      if (kContinuous) reward += 100;
    }
    s.v[0] = pos; s.v[1] = vel;
    so.reward = (float)reward;
  }
  static __device__ __forceinline__ void write_obs(const StateView& sv, const OutView& ov,
                                                   int64_t row,
                                                   const State& s, const StepOut&) {
    if (!ov.env[0]) return;
    static_cast<float2*>(ov.env[0])[row] = make_float2((float)s.v[0], (float)s.v[1]);
  }
};

template <typename R>
using MountainCarDiscrete = MountainCar<R, false>;
template <typename R>
using MountainCarContinuous = MountainCar<R, true>;

// The kernels of Env<float> in f32 mode, of Env<double> otherwise.
template <template <typename> class Env>
KindLaunch classic_launch(int precision, int) {
  return precision == EPB_PREC_F32 ? kind_launch<Env<float>>() : kind_launch<Env<double>>();
}
template <template <typename> class Env>
constexpr int kReals = kStateWords<Env<float>>;

constexpr EnvKey kContinuousAction = {"action", EPB_F32, 1, {1}};

// Pendulum's iopt is its version, which none of its kernels reads.
const KindDesc kClassicKinds[] = {
    {.kind = EPB_CARTPOLE, .keys = {{"obs", EPB_F32, 1, {4}}}, .action = kDiscreteAction,
     .NR = kReals<CartPole>, .launch = classic_launch<CartPole>},
    {.kind = EPB_PENDULUM, .keys = {{"obs", EPB_F32, 1, {3}}}, .action = kContinuousAction,
     .NR = kReals<Pendulum>, .launch = classic_launch<Pendulum>},
    {.kind = EPB_ACROBOT, .keys = {{"obs", EPB_F32, 1, {6}}, {"info:state", EPB_F32, 1, {2}}},
     .action = kDiscreteAction, .NR = kReals<Acrobot>, .launch = classic_launch<Acrobot>},
    {.kind = EPB_MOUNTAIN_CAR, .keys = {{"obs", EPB_F32, 1, {2}}}, .action = kDiscreteAction,
     .NR = kReals<MountainCarDiscrete>, .launch = classic_launch<MountainCarDiscrete>},
    {.kind = EPB_MOUNTAIN_CAR_CONTINUOUS, .keys = {{"obs", EPB_F32, 1, {2}}},
     .action = kContinuousAction, .NR = kReals<MountainCarContinuous>,
     .launch = classic_launch<MountainCarContinuous>},
};
const KindDesc* classic_kind(int kind) { return find_kind(kClassicKinds, kind); }

}  // namespace epb
