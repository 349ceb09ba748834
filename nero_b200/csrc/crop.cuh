// The region crop of the offline tools: a point is kept when it lies in the sphere and / or the box given, tested in fp64
// without contraction so that the numpy oracles reproduce it bit for bit.
#pragma once
#include <cmath>

#include <cuda_runtime.h>

namespace nero {

struct Crop {
  int sphere, box;
  double c[3], r2, lo[3], hi[3];
};

__device__ __forceinline__ bool inside(const Crop& q, double x, double y, double z) {
  if (q.sphere) {
    const double dx = __dsub_rn(x, q.c[0]), dy = __dsub_rn(y, q.c[1]), dz = __dsub_rn(z, q.c[2]);
    if (!(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) <= q.r2)) return false;
  }
  if (q.box) {
    if (!(x >= q.lo[0] && x <= q.hi[0] && y >= q.lo[1] && y <= q.hi[1] && z >= q.lo[2] && z <= q.hi[2])) return false;
  }
  return true;
}

// The crop of sphere (cx, cy, cz, r) and box (lo[3], hi[3]), either of which may be null (no test).  False on bad input: a
// centre or radius that is not finite, r <= 0, or lo > hi (or NaN) on some axis.
inline bool make_crop(const double* sphere, const double* box, Crop& q) {
  q = Crop{};
  if (sphere) {
    for (int a = 0; a < 4; ++a)
      if (!std::isfinite(sphere[a])) return false;
    if (!(sphere[3] > 0.0)) return false;
    q.sphere = 1;
    q.c[0] = sphere[0]; q.c[1] = sphere[1]; q.c[2] = sphere[2];
    q.r2 = sphere[3] * sphere[3];
  }
  if (box) {
    for (int a = 0; a < 3; ++a) {
      if (!(box[a] <= box[3 + a])) return false;
      q.lo[a] = box[a];
      q.hi[a] = box[3 + a];
    }
    q.box = 1;
  }
  return true;
}

}  // namespace nero
