// TEST INFRASTRUCTURE ONLY.  The toolchain's own libstdc++ <random> behind a C API for the one
// recipe Jumanji's Game2048 adds to those of std_rng.cc: std::bernoulli_distribution, and the
// random cell of Game2048Env::AddRandomCell, whose index and value both draw from the engine in
// one C++17 assignment.  tests/test_game2048.py loads crafted engine states into this and into
// the C restatement (oracle/g2048_oracle.c) and compares draw by draw.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <random>
#include <vector>

namespace {
// libstdc++'s mersenne_twister_engine is { _UIntType _M_x[624]; size_t _M_p; } (bits/random.h):
// the state is loaded through the object representation, as std_rng.cc does (this .so must not
// use iostreams inside a host process that has its own).  The seeded-stream test guards it.
struct MtLayout {
  std::mt19937::result_type x[624];
  std::size_t p;
};
static_assert(sizeof(std::mt19937) == sizeof(MtLayout), "unexpected std::mt19937 layout");
}  // namespace

extern "C" {

void* g2s_create() { return new std::mt19937(5489u); }
void g2s_destroy(void* h) { delete static_cast<std::mt19937*>(h); }
void g2s_set(void* h, const uint32_t* mt624, int idx) {
  MtLayout l;
  for (int i = 0; i < 624; ++i) l.x[i] = mt624[i];
  l.p = static_cast<std::size_t>(idx);
  std::memcpy(h, &l, sizeof(l));
}
uint32_t g2s_next(void* h) { return (*static_cast<std::mt19937*>(h))(); }
int g2s_bernoulli(void* h, double prob) {
  std::bernoulli_distribution d(prob);
  return d(*static_cast<std::mt19937*>(h)) ? 1 : 0;
}
// The random cell on a board of n_empty empty cells, written as one assignment whose index and
// value both draw: the right operand is sequenced before the left, so the value comes first.
// Writes the value (2 or 1) and the position among the empty cells.
void g2s_random_cell(void* h, int n_empty, int* value, int* position) {
  auto& gen = *static_cast<std::mt19937*>(h);
  std::vector<int> cells(n_empty, 0);
  std::uniform_int_distribution<int> pick(0, n_empty - 1);
  std::bernoulli_distribution two(0.1);
  cells[pick(gen)] = two(gen) ? 2 : 1;
  for (int i = 0; i < n_empty; ++i)
    if (cells[i] != 0) {
      *value = cells[i];
      *position = i;
    }
}

}  // extern "C"
