// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// Thin C driver around the *unmodified* Jumanji Game2048 header of an envpool checkout
// (envpool/jumanji/game2048_env.h, compiled where it lies; no reference source is copied into
// this repo).  It instantiates the reference's own AsyncEnvPool<Game2048Env> in sync mode and
// exposes Reset / Send+Recv through a flat C ABI, so that oracle/g2048_lib.py can record the
// fixtures in tests/golden/game2048/, pin the C restatement (oracle/g2048_oracle.c) and time the
// reference's thread pool (profiles/game2048_rate.py).  Same drive pattern as ref_driver.cc.
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
#include "envpool/jumanji/game2048_env.h"

namespace {

struct G2048Ref {
  using Pool = jumanji::Game2048EnvPool;
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
  explicit G2048Ref(const Config& config)
      : ids(MakeIds(config["num_envs"_])), num_envs(config["num_envs"_]) {
    spec = std::make_unique<Pool::Spec>(config);
    pool = std::make_unique<Pool>(*spec);
    for (int i = 0; i < num_envs; ++i) ids[i] = i;
  }
  std::vector<Array> MakeAction(const int32_t* action) {
    ::Spec<int> act_spec(std::vector<int>{num_envs});
    Array act(act_spec);
    std::memcpy(act.Data(), action, sizeof(int32_t) * num_envs);
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

// add_random_cell, initial_board and replay_boards are the env's three config keys
// (game2048_add_random_cell, game2048_initial_board, game2048_replay_boards).
// num_threads 0 = the reference's default (hardware concurrency).
void* g2r_create(int num_envs, int num_threads, int seed, int max_episode_steps,
                 int add_random_cell, const char* initial_board, const char* replay_boards) {
  try {
    auto config = G2048Ref::Pool::Spec::kDefaultConfig;
    config["num_envs"_] = num_envs;
    config["batch_size"_] = num_envs;
    config["num_threads"_] = num_threads;
    config["seed"_] = seed;
    if (max_episode_steps > 0) config["max_episode_steps"_] = max_episode_steps;
    config["game2048_add_random_cell"_] = add_random_cell != 0;
    config["game2048_initial_board"_] = std::string(initial_board ? initial_board : "");
    config["game2048_replay_boards"_] = std::string(replay_boards ? replay_boards : "");
    return new G2048Ref(config);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "g2r_create: %s\n", e.what());
    return nullptr;
  }
}
void g2r_destroy(void* h) { delete static_cast<G2048Ref*>(h); }
void g2r_reset(void* h) { static_cast<G2048Ref*>(h)->Reset(); }
void g2r_step(void* h, const int32_t* action) { static_cast<G2048Ref*>(h)->Step(action); }
int g2r_num_keys(void* h) { return static_cast<int>(static_cast<G2048Ref*>(h)->last.size()); }
std::uint64_t g2r_key_bytes(void* h, int k) {
  const Array& a = static_cast<G2048Ref*>(h)->last[k];
  return a.size * a.element_size;
}
void g2r_copy(void* h, int k, void* dst) {
  const Array& a = static_cast<G2048Ref*>(h)->last[k];
  std::memcpy(dst, a.Data(), a.size * a.element_size);
}
// Seconds for `steps` timed Send/Recv pairs after a reset and `warmup` untimed ones; actions
// cycle through a [steps_in_stream, num_envs] stream.
double g2r_bench(void* h, const int32_t* actions, int steps_in_stream, int warmup, int steps) {
  auto* r = static_cast<G2048Ref*>(h);
  r->Reset();
  for (int t = 0; t < warmup; ++t)
    r->Step(actions + static_cast<std::size_t>(t % steps_in_stream) * r->num_envs);
  auto t0 = std::chrono::steady_clock::now();
  for (int t = 0; t < steps; ++t)
    r->Step(actions + static_cast<std::size_t>((warmup + t) % steps_in_stream) * r->num_envs);
  std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
  return dt.count();
}
int g2r_hardware_concurrency() { return static_cast<int>(std::thread::hardware_concurrency()); }

}  // extern "C"
