// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// Thin C driver around the *unmodified* Jumanji Minesweeper header of an envpool checkout
// (envpool/jumanji/minesweeper_env.h, compiled where it lies; no reference source is copied into
// this repo).  It instantiates the reference's own AsyncEnvPool<MinesweeperEnv> in sync mode and
// exposes Reset / Send+Recv through a flat C ABI, so that oracle/ms_lib.py can record the
// fixtures in tests/golden/minesweeper/, pin the C restatement (oracle/ms_oracle.c) and time the
// reference's thread pool (profiles/minesweeper_rate.py).  Same drive pattern as g2048_driver.cc,
// with an action of two int32 (row, column) per env.
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "envpool/core/async_envpool.h"
#include "envpool/jumanji/minesweeper_env.h"

namespace {

struct MsRef {
  using Pool = jumanji::MinesweeperEnvPool;
  std::unique_ptr<Pool::Spec> spec;
  std::unique_ptr<Pool> pool;
  std::vector<Array> last;
  Array ids;
  int num_envs;

  static Array MakeIds(int n) {
    ::Spec<int> s(std::vector<int>{n});
    return Array(s);
  }
  template <typename Config>
  explicit MsRef(const Config& config)
      : ids(MakeIds(config["num_envs"_])), num_envs(config["num_envs"_]) {
    spec = std::make_unique<Pool::Spec>(config);
    pool = std::make_unique<Pool>(*spec);
    for (int i = 0; i < num_envs; ++i) ids[i] = i;
  }
  std::vector<Array> MakeAction(const int32_t* action) {
    ::Spec<int> act_spec(std::vector<int>{num_envs, 2});
    Array act(act_spec);
    std::memcpy(act.Data(), action, sizeof(int32_t) * 2 * num_envs);
    return {ids, ids, act};
  }
  void Reset() {
    pool->Reset(ids);
    last = pool->Recv();
  }
  void Step(const int32_t* action) {
    pool->Send(MakeAction(action));
    last = pool->Recv();
  }
};

}  // namespace

extern "C" {

// The four strings are the env's config keys minesweeper_mine_locations,
// minesweeper_replay_boards, minesweeper_replay_rewards and minesweeper_replay_done.
// num_threads 0 = the reference's default (hardware concurrency).
void* msr_create(int num_envs, int num_threads, int seed, int max_episode_steps,
                 const char* mine_locations, const char* replay_boards,
                 const char* replay_rewards, const char* replay_done) {
  try {
    auto config = MsRef::Pool::Spec::kDefaultConfig;
    config["num_envs"_] = num_envs;
    config["batch_size"_] = num_envs;
    config["num_threads"_] = num_threads;
    config["seed"_] = seed;
    if (max_episode_steps > 0) config["max_episode_steps"_] = max_episode_steps;
    config["minesweeper_mine_locations"_] = std::string(mine_locations ? mine_locations : "");
    config["minesweeper_replay_boards"_] = std::string(replay_boards ? replay_boards : "");
    config["minesweeper_replay_rewards"_] = std::string(replay_rewards ? replay_rewards : "");
    config["minesweeper_replay_done"_] = std::string(replay_done ? replay_done : "");
    return new MsRef(config);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "msr_create: %s\n", e.what());
    return nullptr;
  }
}
void msr_destroy(void* h) { delete static_cast<MsRef*>(h); }
void msr_reset(void* h) { static_cast<MsRef*>(h)->Reset(); }
void msr_step(void* h, const int32_t* action) { static_cast<MsRef*>(h)->Step(action); }
int msr_num_keys(void* h) { return static_cast<int>(static_cast<MsRef*>(h)->last.size()); }
std::uint64_t msr_key_bytes(void* h, int k) {
  const Array& a = static_cast<MsRef*>(h)->last[k];
  return a.size * a.element_size;
}
void msr_copy(void* h, int k, void* dst) {
  const Array& a = static_cast<MsRef*>(h)->last[k];
  std::memcpy(dst, a.Data(), a.size * a.element_size);
}
// Seconds for `steps` timed Send/Recv pairs after a reset and `warmup` untimed ones; actions
// cycle through a [steps_in_stream, num_envs, 2] stream.
double msr_bench(void* h, const int32_t* actions, int steps_in_stream, int warmup, int steps) {
  auto* r = static_cast<MsRef*>(h);
  const std::size_t row = static_cast<std::size_t>(r->num_envs) * 2;
  r->Reset();
  for (int t = 0; t < warmup; ++t) r->Step(actions + static_cast<std::size_t>(t % steps_in_stream) * row);
  auto t0 = std::chrono::steady_clock::now();
  for (int t = 0; t < steps; ++t)
    r->Step(actions + static_cast<std::size_t>((warmup + t) % steps_in_stream) * row);
  std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
  return dt.count();
}
int msr_hardware_concurrency() { return static_cast<int>(std::thread::hardware_concurrency()); }

}  // extern "C"
