// boxmuller.cuh -- the standard normals of the throughput-mode streams (device only): two per
// Philox block, u = u01(x, y) for the radius and v = u01(z, w) for the angle.
#pragma once

#include "philox.cuh"

namespace elfi {

// two standard normals from one Philox block (Box-Muller)
__device__ __forceinline__ void normal2(const uint4& r, double& n0, double& n1) {
    const double u = u01(r.x, r.y), v = u01(r.z, r.w);
    const double rad = sqrt(-2.0 * log(u));
    double s, c;
    sincospi(2.0 * v, &s, &c);
    n0 = rad * c;
    n1 = rad * s;
}

}  // namespace elfi
