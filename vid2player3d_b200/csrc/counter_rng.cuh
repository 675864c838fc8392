// Counter-based random numbers shared by the env launches: a draw is a pure function of (seed, launch counter, index), so a
// launch that keeps its counter in device memory draws fresh numbers on every replay of a CUDA graph and needs no RNG launch.
#pragma once
#include <stdint.h>

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// the 64 random bits of draw idx of launch `counter`
__device__ __forceinline__ uint64_t counter_bits(uint64_t seed, uint64_t counter, uint64_t idx) {
  return splitmix64(splitmix64(seed ^ (counter * 0xD1B54A32D192ED03ull)) + idx);
}
