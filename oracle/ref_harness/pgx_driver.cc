// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// Thin C driver around the *unmodified* PGX board-game header of an envpool checkout
// (envpool/pgx/board_games.h, compiled where it lies; no reference source is copied into this
// repo).  It instantiates the reference's own AsyncEnvPool<TicTacToeEnv> or
// AsyncEnvPool<ConnectFourEnv> with max_num_players = 2, batch_size = num_envs and one worker
// thread, and exposes Reset / Send+Recv through a flat C ABI, so that oracle/pgx_lib.py can record
// the fixtures in tests/golden/pgx/, pin the C restatement (oracle/pgx_oracle.c) and time the
// reference's thread pool (profiles/pgx_rate.py).  A multi-player pool never runs in the
// reference's sync mode (async_envpool.h:97): rows come back in completion order, which with one
// worker thread is submission order.  Each step takes explicit env_id and players.env_id rows, so
// permuted or duplicated player rows reach the reference's own ParseAction.
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
#include "envpool/pgx/board_games.h"

namespace {

struct PgxRefBase {
  virtual ~PgxRefBase() = default;
  virtual void Reset() = 0;
  virtual void Step(const int32_t* env_id, int n, const int32_t* players_env_id,
                    const int32_t* action, int m) = 0;
  std::vector<Array> last;
  int num_envs = 0;
};

template <typename Pool>
struct PgxRef : PgxRefBase {
  std::unique_ptr<typename Pool::Spec> spec;
  std::unique_ptr<Pool> pool;

  static Array IntArray(int n, const int32_t* v) {
    ::Spec<int> s(std::vector<int>{n});
    Array a(s);
    std::memcpy(a.Data(), v, sizeof(int32_t) * n);
    return a;
  }
  PgxRef(int n, int num_threads, int seed) {
    auto config = Pool::Spec::kDefaultConfig;
    config["num_envs"_] = n;
    config["batch_size"_] = n;
    config["num_threads"_] = num_threads;
    config["max_num_players"_] = 2;
    config["seed"_] = seed;
    spec = std::make_unique<typename Pool::Spec>(config);
    pool = std::make_unique<Pool>(*spec);
    num_envs = n;
  }
  void Reset() override {
    std::vector<int32_t> ids(num_envs);
    for (int i = 0; i < num_envs; ++i) ids[i] = i;
    pool->Reset(IntArray(num_envs, ids.data()));
    last = pool->Recv();
  }
  void Step(const int32_t* env_id, int n, const int32_t* players_env_id, const int32_t* action,
            int m) override {
    pool->Send(std::vector<Array>{IntArray(n, env_id), IntArray(m, players_env_id),
                                  IntArray(m, action)});
    last = pool->Recv();
  }
};

}  // namespace

extern "C" {

// game 0 = TicTacToe, 1 = ConnectFour.  num_threads 0 = the reference's default (hardware
// concurrency); row order is submission order only with 1.
void* pgr_create(int game, int num_envs, int num_threads, int seed) {
  try {
    if (game == 0) return new PgxRef<pgx::TicTacToeEnvPool>(num_envs, num_threads, seed);
    if (game == 1) return new PgxRef<pgx::ConnectFourEnvPool>(num_envs, num_threads, seed);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "pgr_create: %s\n", e.what());
  }
  return nullptr;
}
void pgr_destroy(void* h) { delete static_cast<PgxRefBase*>(h); }
void pgr_reset(void* h) { static_cast<PgxRefBase*>(h)->Reset(); }
// Every env must own at least one players.env_id row (the reference reads a zero-length array
// otherwise).  batch_size = num_envs, so n must be num_envs.
void pgr_step(void* h, const int32_t* env_id, int n, const int32_t* players_env_id,
              const int32_t* action, int m) {
  static_cast<PgxRefBase*>(h)->Step(env_id, n, players_env_id, action, m);
}
int pgr_num_keys(void* h) { return static_cast<int>(static_cast<PgxRefBase*>(h)->last.size()); }
std::uint64_t pgr_key_bytes(void* h, int k) {
  const Array& a = static_cast<PgxRefBase*>(h)->last[k];
  return a.size * a.element_size;
}
void pgr_copy(void* h, int k, void* dst) {
  const Array& a = static_cast<PgxRefBase*>(h)->last[k];
  std::memcpy(dst, a.Data(), a.size * a.element_size);
}
// Seconds for `steps` timed Send/Recv pairs after a reset and `warmup` untimed ones; one action
// per env (players.env_id = env_id), cycling through a [steps_in_stream, num_envs] stream.
double pgr_bench(void* h, const int32_t* actions, int steps_in_stream, int warmup, int steps) {
  auto* r = static_cast<PgxRefBase*>(h);
  const std::size_t row = static_cast<std::size_t>(r->num_envs);
  std::vector<int32_t> ids(r->num_envs);
  for (int i = 0; i < r->num_envs; ++i) ids[i] = i;
  auto step = [&](int t) {
    r->Step(ids.data(), r->num_envs, ids.data(),
            actions + static_cast<std::size_t>(t % steps_in_stream) * row, r->num_envs);
  };
  r->Reset();
  for (int t = 0; t < warmup; ++t) step(t);
  auto t0 = std::chrono::steady_clock::now();
  for (int t = 0; t < steps; ++t) step(warmup + t);
  std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
  return dt.count();
}
int pgr_hardware_concurrency() { return static_cast<int>(std::thread::hardware_concurrency()); }

}  // extern "C"
