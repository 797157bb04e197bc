// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// pgx_driver.cc's driver (compiled in here, unchanged) for the reference's own
// AsyncEnvPool<HexEnv> and AsyncEnvPool<OthelloEnv> from the *unmodified* PGX board-game header
// of an envpool checkout.  The pool is created by pgr_create_hex_othello; every other entry
// point (pgr_step, pgr_copy, pgr_bench, ...) is pgx_driver.cc's, in this library's own copy.
// oracle/hex_othello_lib.py loads it as _ref/libhex_othello_ref.so.
#include "pgx_driver.cc"

extern "C" {

// game 0 = Hex, 1 = Othello; the other arguments as pgr_create's
void* pgr_create_hex_othello(int game, int num_envs, int num_threads, int seed) {
  try {
    if (game == 0) return new PgxRef<pgx::HexEnvPool>(num_envs, num_threads, seed);
    if (game == 1) return new PgxRef<pgx::OthelloEnvPool>(num_envs, num_threads, seed);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "pgr_create_hex_othello: %s\n", e.what());
  }
  return nullptr;
}

}  // extern "C"
