// TEST INFRASTRUCTURE ONLY.  The toolchain's own libstdc++ behind a C API for the one recipe
// Jumanji's Minesweeper adds to those of std_rng.cc: std::shuffle of iota(100) on a std::mt19937,
// as MinesweeperEnv::Reset places random mines.  tests/test_minesweeper.py loads crafted engine
// states into this, into the C restatement (oracle/ms_oracle.c) and into a model of the kernel's
// register-only shuffle, and compares the permutations and the engine positions after them.
#include <algorithm>
#include <array>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <random>

namespace {
// libstdc++'s mersenne_twister_engine is { _UIntType _M_x[624]; size_t _M_p; } (bits/random.h),
// loaded through the object representation as std_rng.cc and g2048_std_rng.cc do.
struct MtLayout {
  std::mt19937::result_type x[624];
  std::size_t p;
};
static_assert(sizeof(std::mt19937) == sizeof(MtLayout), "unexpected std::mt19937 layout");
}  // namespace

extern "C" {

void* mss_create() { return new std::mt19937(5489u); }
void mss_destroy(void* h) { delete static_cast<std::mt19937*>(h); }
void mss_set(void* h, const uint32_t* mt624, int idx) {
  MtLayout l;
  for (int i = 0; i < 624; ++i) l.x[i] = mt624[i];
  l.p = static_cast<std::size_t>(idx);
  std::memcpy(h, &l, sizeof(l));
}
uint32_t mss_next(void* h) { return (*static_cast<std::mt19937*>(h))(); }
void mss_shuffle(void* h, int32_t* out100) {
  std::array<int, 100> locations{};
  std::iota(locations.begin(), locations.end(), 0);
  std::shuffle(locations.begin(), locations.end(), *static_cast<std::mt19937*>(h));
  for (int i = 0; i < 100; ++i) out100[i] = locations[i];
}

}  // extern "C"
