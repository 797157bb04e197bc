// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// pgx_driver.cc's driver (compiled in here, unchanged) for the reference's own
// AsyncEnvPool<ChessEnv> and AsyncEnvPool<GardnerChessEnv> from the *unmodified* PGX chess header
// of an envpool checkout (envpool/pgx/chess_games.h).  The pool is created by pgr_create_chess;
// every other entry point (pgr_step, pgr_copy, pgr_bench, ...) is pgx_driver.cc's, in this
// library's own copy.  oracle/chess_lib.py loads it as _ref/libchess_ref.so.
#include "pgx_driver.cc"
#include "envpool/pgx/chess_games.h"

extern "C" {

// game 0 = Chess, 1 = GardnerChess; the rest as pgr_create's
void* pgr_create_chess(int game, int num_envs, int num_threads, int seed) {
  try {
    if (game == 0) return new PgxRef<pgx::ChessEnvPool>(num_envs, num_threads, seed);
    if (game == 1) return new PgxRef<pgx::GardnerChessEnvPool>(num_envs, num_threads, seed);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "pgr_create_chess: %s\n", e.what());
  }
  return nullptr;
}

}  // extern "C"
