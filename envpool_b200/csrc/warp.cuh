// Warp-cooperative helpers of the one-warp-per-env kernels (go.cu, chess.cu).
#pragma once

#include <cstdint>

namespace epb {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// A warp writes n bytes at dst (any alignment), byte i = f(i): 4-byte stores in the middle.
template <class F>
__device__ __forceinline__ void warp_write_bytes(uint8_t* dst, int n, int lane, F f) {
  int head = (int)((4u - ((uint32_t)(uintptr_t)dst & 3u)) & 3u);
  head = head < n ? head : n;
  if (lane < head) dst[lane] = f(lane);
  const int words = (n - head) >> 2;
  uint32_t* w = reinterpret_cast<uint32_t*>(dst + head);
  for (int i = lane; i < words; i += 32) {
    const int b = head + 4 * i;
    w[i] = (uint32_t)f(b) | ((uint32_t)f(b + 1) << 8) | ((uint32_t)f(b + 2) << 16) |
           ((uint32_t)f(b + 3) << 24);
  }
  const int tail0 = head + 4 * words;
  if (tail0 + lane < n) dst[tail0 + lane] = f(tail0 + lane);
}

}  // namespace epb
