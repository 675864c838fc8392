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

// N(0, 1) draw idx of launch `step`: Box-Muller on two 24-bit fields of counter_bits.  u1 lies in (0, 1), so the log is finite and
// |result| <= sqrt(48 ln 2) ~ 5.77.
__device__ __forceinline__ float counter_normal(uint64_t seed, uint64_t step, uint64_t idx) {
  const uint64_t h = counter_bits(seed, step, idx);
  const float u1 = ((uint32_t)(h >> 40) + 1u) * (1.0f / 16777217.0f);     // (0, 1)
  const float u2 = (uint32_t)((h >> 8) & 0xFFFFFFu) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
}

// the last block of the grid to get here adds inc to the device counter and re-arms the done ticket, so the next launch (a CUDA
// graph replay included) draws with the next counter value.  Every thread of the block must call it; a block may call it from two
// places (e.g. a warp-specialised kernel's producer and consumer branches), since each thread passes its two barriers once.
__device__ __forceinline__ void last_block_advance(int64_t* counter, unsigned int* done, int64_t inc) {
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (last && threadIdx.x == 0) { counter[0] += inc; *done = 0u; __threadfence(); }
}
