// The counter hash every random draw of libsvpointops comes from: a value of (seed, a, b), reproducible and independent of
// launch order, with nothing stored between calls.
#pragma once

namespace sv {

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}
__device__ __forceinline__ unsigned hash_u32(unsigned long long seed, unsigned long long a, unsigned long long b) {
  return (unsigned)(mix64(seed + a * 0x9E3779B97F4A7C15ULL + mix64(b + 0xD1B54A32D192ED03ULL)) >> 16);
}

}  // namespace sv
