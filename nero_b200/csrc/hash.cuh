// Counter-based random numbers shared by the relighting path tracer (math_relight.cuh) and the surface sampler
// (k_meshpts.cu).  Host+device, so tests/hostcheck compiles the same expression for the CPU; the oracles restate it in numpy.
#pragma once
#include <cstdint>

#include "common.cuh"

namespace nero {

NERO_HD uint32_t rl_mix(uint32_t x) {     // murmur3 finaliser
  x ^= x >> 16; x *= 0x85ebca6bu;
  x ^= x >> 13; x *= 0xc2b2ae35u;
  x ^= x >> 16;
  return x;
}

}  // namespace nero
