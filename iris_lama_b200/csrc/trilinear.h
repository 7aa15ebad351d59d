// trilinear.h -- the trilinear interpolation of the 3-D distance queries, shared by TruncatedSignedDistanceMap (tsdm_core.h,
// truncated_signed_distance_map.cpp:59-130) and DynamicDistanceMap (ddm3_core.h, dynamic_distance_map.cpp:93-133), whose is_3d
// branches have the same form.  Every rounding step is spelled out (mul_rn / add_rn, no contraction), so the device and a host run
// agree bit for bit.  Plain C++ usable from host and device.
#pragma once

#include "lama_core.h"

namespace lama_b200 {

// The cell c = (uint32) w2m_nocast(pt) and the fractions mu = m - c, nu = 1 - mu of a world point
LAMA_HD void cell_fraction(const double pt[3], double scale, uint32_t c[3], double mu[3], double nu[3])
{
    for (int k = 0; k < 3; ++k) {
        const double m = w2m_nocast(pt[k], scale);
        c[k] = (uint32_t)m;
        mu[k] = add_rn(m, -(double)c[k]);
        nu[k] = add_rn(1.0, -mu[k]);
    }
}

// distance(Vector3d, gradient) in 3-D: `value(x, y, z)` is the map's distance(Vector3ui) at the 8 corners V000 V100 V010 V110 V001 ...
template <class Value>
LAMA_HD double trilinear_distance(const double pt[3], double scale, Value&& value, double grad[3])
{
    double mu[3], nu[3];
    uint32_t c[3];
    cell_fraction(pt, scale, c, mu, nu);
    double v[8];
    for (int i = 0; i < 8; ++i) v[i] = value(c[0] + (i & 1), c[1] + ((i >> 1) & 1), c[2] + (i >> 2));
    const double dist =
        add_rn(add_rn(add_rn(add_rn(add_rn(add_rn(add_rn(
            mul_rn(v[0], mul_rn(mul_rn(nu[0], nu[1]), nu[2])),
            mul_rn(mul_rn(mul_rn(v[1], mu[0]), nu[1]), nu[2])),
            mul_rn(mul_rn(mul_rn(v[2], nu[0]), mu[1]), nu[2])),
            mul_rn(mul_rn(mul_rn(v[3], mu[0]), mu[1]), nu[2])),
            mul_rn(mul_rn(mul_rn(v[4], nu[0]), nu[1]), mu[2])),
            mul_rn(mul_rn(mul_rn(v[5], mu[0]), nu[1]), mu[2])),
            mul_rn(mul_rn(mul_rn(v[6], nu[0]), mu[1]), mu[2])),
            mul_rn(v[7], mul_rn(mul_rn(mu[0], mu[1]), mu[2])));
    double a, b;
    a = add_rn(mul_rn(add_rn(v[0], -v[1]), nu[1]), mul_rn(add_rn(v[2], -v[3]), mu[1]));
    b = add_rn(mul_rn(add_rn(v[4], -v[5]), nu[1]), mul_rn(add_rn(v[6], -v[7]), mu[1]));
    grad[0] = mul_rn(-add_rn(mul_rn(a, nu[2]), mul_rn(b, mu[2])), scale);
    a = add_rn(mul_rn(add_rn(v[0], -v[2]), nu[0]), mul_rn(add_rn(v[1], -v[3]), mu[0]));
    b = add_rn(mul_rn(add_rn(v[4], -v[6]), nu[0]), mul_rn(add_rn(v[5], -v[7]), mu[0]));
    grad[1] = mul_rn(-add_rn(mul_rn(a, nu[2]), mul_rn(b, mu[2])), scale);
    a = add_rn(mul_rn(add_rn(v[0], -v[4]), nu[0]), mul_rn(add_rn(v[1], -v[5]), mu[0]));
    b = add_rn(mul_rn(add_rn(v[2], -v[6]), nu[0]), mul_rn(add_rn(v[3], -v[7]), mu[0]));
    grad[2] = mul_rn(-add_rn(mul_rn(a, nu[1]), mul_rn(b, mu[1])), scale);
    return dist;
}

}  // namespace lama_b200
