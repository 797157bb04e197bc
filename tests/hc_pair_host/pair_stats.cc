// Test / profiling infrastructure: the host build of the pair-lane HalfCheetah algorithm with its
// solver branch trace (HCP_STATS, envpool_b200/csrc/mujoco_pair.cuh).  Each lane appends the
// (event, value) pairs of the branches its solver takes to its own trace; the CPU suite
// (tests/hc_solver_cases.py) reads both, profiles/hc_pair_iteration_stats.py summarises them.
#define HCP_HOST 1
#define HCP_STATS 1
#include <barrier>
#include <cstring>
#include <thread>
#include <vector>

static std::vector<int> g_trace[2];  // per lane: event, value, event, value, ...
static double g_smooth[9];           // qacc_smooth of the last mj_step
static void hcp_trace(int side, int ev, int val) {
  g_trace[side].push_back(ev);
  g_trace[side].push_back(val);
}
static void hcp_trace_smooth(int side, const double* r, const double* l) {
  for (int i = 0; i < 3; ++i) {
    if (side == 0) g_smooth[i] = r[i];
    g_smooth[3 + 3 * side + i] = l[i];
  }
}

#include "../../envpool_b200/csrc/mujoco_pair.cuh"

namespace epb {
namespace hcp {

struct Chan {
  std::barrier<> bar{2};
  double slot[2];
};

double host_xch(void* chan, int side, double v) {
  Chan* ch = static_cast<Chan*>(chan);
  ch->slot[side] = v;
  ch->bar.arrive_and_wait();
  const double r = ch->slot[side ^ 1];
  ch->bar.arrive_and_wait();
  return r;
}

}  // namespace hcp
}  // namespace epb

using namespace epb;

// Forget both lanes' traces.
extern "C" void hc_pair_trace_clear() {
  g_trace[0].clear();
  g_trace[1].clear();
}

// Copies at most `cap` ints of lane `side`'s trace to `out`; returns the trace's length.
extern "C" int hc_pair_trace(int side, int* out, int cap) {
  const int n = (int)g_trace[side].size();
  std::memcpy(out, g_trace[side].data(), sizeof(int) * (n < cap ? n : cap));
  return n;
}

// qacc_smooth [9] of the last mj_step.
extern "C" void hc_pair_last_smooth(double* out) { std::memcpy(out, g_smooth, sizeof g_smooth); }

// As hc_pair_host_step in pair_host.cc: nsub mj_steps of one env, state updated in place.
extern "C" int hc_pair_host_step(const void* model_blob, double* q, double* v, double* w,
                                 const double* ctrl, int nsub, int ks) {
  hcm::HcModel cm;
  std::memcpy(&cm, model_blob, sizeof(cm));
  hcm::LegModel lm[2];
  hcm::leg_model_of(cm, 0, &lm[0]);
  hcm::leg_model_of(cm, 1, &lm[1]);
  hcp::Chan chan;
  hcp::PairState st[2];
  auto lane = [&](int side) {
    hcp::PairState& s = st[side];
    const int l0 = 3 + 3 * side;
    for (int i = 0; i < 3; ++i) {
      s.qr[i] = q[i]; s.vr[i] = v[i]; s.wr[i] = w[i];
      s.ql[i] = q[l0 + i]; s.vl[i] = v[l0 + i]; s.wl[i] = w[l0 + i];
      s.ctrl[i] = ctrl[3 * side + i];
    }
    double srow[hcp::MAXR * hcp::NF], ovf[hcp::MAXR * hcp::NF];
    hcp::Ctx c;
    c.side = side; c.pm = 0; c.chan = &chan;
    c.srow = srow; c.ks = ks; c.ovf = ovf;
    for (int k = 0; k < nsub; ++k) hcp::pair_substep(c, cm, lm[side], s);
  };
  std::thread t1(lane, 1);
  lane(0);
  t1.join();
  int bad = 0;
  for (int i = 0; i < 3; ++i) {
    bad |= std::memcmp(&st[0].qr[i], &st[1].qr[i], 8) != 0;
    bad |= std::memcmp(&st[0].vr[i], &st[1].vr[i], 8) != 0;
    bad |= std::memcmp(&st[0].wr[i], &st[1].wr[i], 8) != 0;
    q[i] = st[0].qr[i]; v[i] = st[0].vr[i]; w[i] = st[0].wr[i];
    q[3 + i] = st[0].ql[i]; v[3 + i] = st[0].vl[i]; w[3 + i] = st[0].wl[i];
    q[6 + i] = st[1].ql[i]; v[6 + i] = st[1].vl[i]; w[6 + i] = st[1].wl[i];
  }
  return bad;
}
