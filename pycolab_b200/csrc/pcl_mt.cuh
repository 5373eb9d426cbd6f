// pcl_mt.cuh — MT19937, warp-cooperative, bit-compatible with NumPy's legacy
// RandomState and with Python's `random` module (both are MT19937 over a 624-word
// key + position; state word 624 is the position).  Used by marauders.cu
// (np.random.choice), shockwave.cu (np.random.randint), apprehend.cu
// (random.uniform), t_maze.cu and compiled.cu (the draws of compiled update() code).
#pragma once

#include <stdint.h>

#include "pcl_device.cuh"

namespace pcl {

// ---- MT19937 (NumPy legacy RandomState core), warp-cooperative ------------
__device__ __forceinline__ void mt_twist(uint32_t* mt, int lane) {
  for (int base = 0; base < 624; base += 32) {
    const int j = base + lane;
    uint32_t v = 0;
    if (j < 624) {
      const int j1 = (j + 1 == 624) ? 0 : j + 1;
      const int jm = (j + 397 >= 624) ? j + 397 - 624 : j + 397;
      const uint32_t y = (mt[j] & 0x80000000u) | (mt[j1] & 0x7fffffffu);
      v = mt[jm] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    __syncwarp();
    if (j < 624) mt[j] = v;
    __syncwarp();
  }
}
// Twist: the twist to run, e.g. an out-of-line copy of mt_twist for a caller that cannot
// afford the registers of an inlined one.
template <void (*Twist)(uint32_t*, int) = mt_twist>
__device__ __forceinline__ uint32_t mt_next(uint32_t* mt, int lane) {
  int pos = (int)mt[624];
  if (pos >= 624) { Twist(mt, lane); pos = 0; }
  uint32_t y = mt[pos];
  __syncwarp();
  if (lane == 0) mt[624] = (uint32_t)(pos + 1);
  __syncwarp();
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}
// RandomState.randint(0, n) for 1 <= n <= 2^32: masked rejection; no draw when
// n == 1.
__device__ __forceinline__ uint32_t mt_below(uint32_t* mt, uint32_t n, int lane) {
  const uint32_t rng = n - 1;
  if (rng == 0) return 0;
  uint32_t mask = rng;
  mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
  uint32_t v;
  do { v = mt_next(mt, lane) & mask; } while (v > rng);
  return v;
}

// The three draws of mt_draw.
enum MtRule {
  kMtNumpyBelow,    // mt_below(n), 1 <= n < 2^32
  kMtPythonBelow,   // Python's Random._randbelow(n), 1 <= n <= 2^32
  kMtRandom53       // the 53 bits of mt_random53 as an integer (n unused)
};

// One draw through a single mt_next call site: every inlined copy of the twist costs its
// caller registers, so an interpreter that offers all three draws calls this once.
//   kMtNumpyBelow: as mt_below.
//   kMtPythonBelow: Lib/random.py _randbelow_with_getrandbits: getrandbits(k),
//     k = n.bit_length(), until it is below n.  getrandbits (Modules/_randommodule.c) is
//     one output >> (32 - k) for k <= 32, and for k == 33 two outputs, least significant
//     word first, the second cut to its top bit.  Unlike NumPy, n == 1 consumes output.
//   kMtRandom53: (a >> 5) << 26 | (b >> 6) of two outputs a, b; times 2^-53 (exact) it
//     is mt_random53's double.
template <void (*Twist)(uint32_t*, int) = mt_twist>
__device__ __forceinline__ uint64_t mt_draw(uint32_t* mt, MtRule rule, uint64_t n, int lane) {
  if (rule == kMtNumpyBelow && n == 1) return 0;
  const int k = 64 - __clzll((long long)(rule == kMtNumpyBelow ? n - 1 : n));
  const uint64_t mask = (1ull << k) - 1;                     // NumPy's gen_mask(n - 1)
  const int words = rule == kMtRandom53 || (rule == kMtPythonBelow && k > 32) ? 2 : 1;
  for (;;) {
    uint32_t first = 0, y = 0;
#pragma unroll 1
    for (int i = 0; i < words; ++i) {
      first = y;
      y = mt_next<Twist>(mt, lane);
    }
    uint64_t r;
    if (rule == kMtRandom53) return (uint64_t)(first >> 5) << 26 | (y >> 6);
    if (rule == kMtNumpyBelow) r = y & mask;
    else r = words == 2 ? (first | (uint64_t)(y >> 31) << 32) : (uint64_t)(y >> (32 - k));
    if (r < n) return r;
  }
}


// Python `random.random()` (Modules/_randommodule.c genrand_res53): 53 random bits
// from two outputs, as an exactly representable double.
__device__ __forceinline__ double mt_random53(uint32_t* mt, int lane) {
  const uint32_t a = mt_next(mt, lane) >> 5, b = mt_next(mt, lane) >> 6;
  return __dmul_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)b),
                   1.0 / 9007199254740992.0);
}

}  // namespace pcl
