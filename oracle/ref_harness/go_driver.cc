// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// pgx_driver.cc's driver (compiled in here, unchanged) for the reference's own
// AsyncEnvPool<GoEnv> from the *unmodified* PGX Go header of an envpool checkout
// (envpool/pgx/go.h), with board_size, komi and max_terminal_steps set.  The pool is created by
// pgr_create_go; every other entry point (pgr_step, pgr_copy, pgr_bench, ...) is pgx_driver.cc's,
// in this library's own copy.  oracle/go_lib.py loads it as _ref/libgo_ref.so.
#include "pgx_driver.cc"
#include "envpool/pgx/go.h"

namespace {

// PgxRef with the Go options in the config: two players, batch_size = num_envs
struct GoRef : PgxRefBase {
  std::unique_ptr<pgx::GoEnvPool::Spec> spec;
  std::unique_ptr<pgx::GoEnvPool> pool;

  GoRef(int size, double komi, int max_terminal_steps, int n, int num_threads, int seed) {
    auto config = pgx::GoEnvPool::Spec::kDefaultConfig;
    config["num_envs"_] = n;
    config["batch_size"_] = n;
    config["num_threads"_] = num_threads;
    config["max_num_players"_] = 2;
    config["seed"_] = seed;
    config["board_size"_] = size;
    config["komi"_] = komi;
    config["max_terminal_steps"_] = max_terminal_steps;
    config["task"_] = std::string("go_") + std::to_string(size) + "x" + std::to_string(size);
    spec = std::make_unique<pgx::GoEnvPool::Spec>(config);
    pool = std::make_unique<pgx::GoEnvPool>(*spec);
    num_envs = n;
  }
  void Reset() override {
    std::vector<int32_t> ids(num_envs);
    for (int i = 0; i < num_envs; ++i) ids[i] = i;
    pool->Reset(PgxRef<pgx::TicTacToeEnvPool>::IntArray(num_envs, ids.data()));
    last = pool->Recv();
  }
  void Step(const int32_t* env_id, int n, const int32_t* players_env_id, const int32_t* action,
            int m) override {
    using R = PgxRef<pgx::TicTacToeEnvPool>;
    pool->Send(std::vector<Array>{R::IntArray(n, env_id), R::IntArray(m, players_env_id),
                                  R::IntArray(m, action)});
    last = pool->Recv();
  }
};

}  // namespace

extern "C" {

// board_size 9, 13 or 19; max_terminal_steps 0 = 2 board_size^2; the rest as pgr_create's
void* pgr_create_go(int size, double komi, int max_terminal_steps, int num_envs, int num_threads,
                    int seed) {
  try {
    return new GoRef(size, komi, max_terminal_steps, num_envs, num_threads, seed);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "pgr_create_go: %s\n", e.what());
  }
  return nullptr;
}

}  // extern "C"
