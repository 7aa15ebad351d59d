// tsdm_core.h -- the arithmetic of lama::TruncatedSignedDistanceMap, shared by the sm_90a kernels (tsdm.cu) and the host
// emulation tests.  Plain C++ usable from host and device.
//
// Reference: include/lama/sdm/truncated_signed_distance_map.h, src/sdm/truncated_signed_distance_map.cpp (integrate :161-208,
// distance :59-139, toMesh :220-272), src/sdm/marching_cubes.cpp (interpolate_vertex, calculate_vertex_configuration),
// Map::computeRay src/sdm/map.cpp:229-258.
//
// Every rounding step of the reference is spelled out: fp64 with mul_rn / add_rn (lama_core.h) where the reference computes in
// double, fp32 with the f*_rn helpers below where it computes in float, and an explicit rounding to float wherever the reference
// stores a double into a float.  No contraction anywhere, so the device cells are bit-identical to a sequential host run.
#pragma once

#include "ray_core.h"
#include "match_core.h"

namespace lama_b200 {

constexpr int kTsdmCells2D = kPatchCells;               // 32 x 32 cells of 8 bytes per patch
constexpr int kTsdmCells3D = kPatchCells * kPatchLen;   // 32 x 32 x 32

#if defined(__CUDA_ARCH__)
LAMA_HD float fadd_rn(float a, float b) { return __fadd_rn(a, b); }
LAMA_HD float fmul_rn(float a, float b) { return __fmul_rn(a, b); }
LAMA_HD float fdiv_rn(float a, float b) { return __fdiv_rn(a, b); }
#else
LAMA_HD float fadd_rn(float a, float b) { volatile float r = a + b; return r; }
LAMA_HD float fmul_rn(float a, float b) { volatile float r = a * b; return r; }
LAMA_HD float fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
#endif

// Map::m2w (map.h:147-148) of one coordinate
LAMA_HD double m2w(uint32_t c, double scale) { return add_rn((double)c, -(double)kMapOffsetCells) / scale; }
// (a0 b0 + a1 b1) + a2 b2: Eigen's squaredNorm / dot of a Vector3d
LAMA_HD double dot3(const double a[3], const double b[3]) { return add_rn(add_rn(mul_rn(a[0], b[0]), mul_rn(a[1], b[1])), mul_rn(a[2], b[2])); }

struct TsdmParams {
    double scale;       // 1 / resolution
    float truncate;     // truncate_size_ (0.15, setMaxDistance)
    float delta;        // delta_ = 4 resolution
    float epsilon;      // epsilon_ = resolution
    float max_weight;   // maximum_weight_ = 10000
    int is3d;
};

// integrate()'s per-ray state (:164-183): the walk ends and the two cached reciprocals
struct TsdmRay {
    double hit[3];
    double oh[3];       // origin_to_hit
    float inv_sq;       // inv_squared_norm
    float inv_de;       // inv_delta_less_epsilon
    BeamCells cells;    // computeRay(start, end), both ends excluded
};

LAMA_HD TsdmRay tsdm_ray(const double origin[3], const double hit[3], const TsdmParams& p)
{
    TsdmRay r;
    double dir[3];
    for (int k = 0; k < 3; ++k) {
        r.hit[k] = hit[k];
        dir[k] = add_rn(hit[k], -origin[k]);
        r.oh[k] = dir[k];
    }
    const double sq = dot3(dir, dir);
    const float squared_norm = (float)sq;
    if (sq > 0.0) {   // Vector3d::normalize
        const double nrm = sqrt(sq);
        for (int k = 0; k < 3; ++k) dir[k] = dir[k] / nrm;
    }
    const float truncate = p.truncate < squared_norm ? p.truncate : squared_norm;   // std::min(squared_norm, truncate_size_)
    for (int k = 0; k < 3; ++k) {
        r.cells.from[k] = w2m(add_rn(hit[k], -mul_rn(dir[k], (double)truncate)), p.scale);
        r.cells.to[k]   = w2m(add_rn(hit[k], mul_rn(dir[k], (double)p.truncate)), p.scale);
    }
    r.cells.mark_hit = true;
    r.inv_sq = (float)(1.0 / (double)squared_norm);
    r.inv_de = (float)(1.0 / (double)fadd_rn(p.delta, -p.epsilon));
    return r;
}

// One voxel of integrate() (:190-205): its signed distance d and weight w; false where the reference `continue`s (d < -delta_).
// The voxel is allocated and "on" either way.
LAMA_HD bool tsdm_sample(const TsdmRay& r, uint32_t cx, uint32_t cy, uint32_t cz, const TsdmParams& p, float& d, float& w)
{
    const double ch[3] = {add_rn(r.hit[0], -m2w(cx, p.scale)), add_rn(r.hit[1], -m2w(cy, p.scale)), add_rn(r.hit[2], -m2w(cz, p.scale))};
    const double norm = sqrt(dot3(ch, ch));
    const double dp = dot3(ch, r.oh);
    const int sg = (0.0 < dp) - (dp < 0.0);
    d = (float)mul_rn(norm, (double)sg);
    if (d < -p.delta) return false;
    if (-p.delta <= d && d <= -p.epsilon) w = fmul_rn(fmul_rn(fadd_rn(d, p.delta), r.inv_sq), r.inv_de);
    else w = r.inv_sq;
    return true;
}

// the running average of :203-204, all float
LAMA_HD void tsdm_fold(float& cd, float& cw, float d, float w, float max_weight)
{
    const float sum = fadd_rn(cw, w);
    cd = fdiv_rn(fadd_rn(fmul_rn(cw, cd), fmul_rn(w, d)), sum);
    cw = max_weight < sum ? max_weight : sum;
}

// ---- directory window of the device store ----------------------------------------------------------------------------------
// dim[0] x dim[1] x dim[2] patches from patch coordinates base (cell >> 5); dim[2] == 1 and z ignored in 2-D (MASK3D, map.h:182-189)
struct TsdmWindow {
    int32_t base[3];
    int32_t dim[3];
    int is3d;
};
// directory index (x fastest, then y, then z), or -1 outside the window
LAMA_HD int tsdm_dir_index(const TsdmWindow& w, uint32_t x, uint32_t y, uint32_t z)
{
    const int px = (int)(x >> kPatchLog2) - w.base[0], py = (int)(y >> kPatchLog2) - w.base[1];
    const int pz = w.is3d ? (int)(z >> kPatchLog2) - w.base[2] : 0;
    if ((unsigned)px >= (unsigned)w.dim[0] || (unsigned)py >= (unsigned)w.dim[1] || (unsigned)pz >= (unsigned)w.dim[2]) return -1;
    return (pz * w.dim[1] + py) * w.dim[0] + px;
}
// Map::m2c (map.h:182-189)
LAMA_HD uint32_t tsdm_cell_index(uint32_t x, uint32_t y, uint32_t z, int is3d)
{
    const uint32_t m = kPatchLen - 1;
    return (x & m) | ((y & m) << kPatchLog2) | (is3d ? (z & m) << (2 * kPatchLog2) : 0u);
}

// ---- queries ---------------------------------------------------------------------------------------------------------------
// distance(Vector3d, gradient) (:59-130).  `value(x, y, z)` is distance(Vector3ui) (:132-139): truncate_size_ for an absent cell or
// one of weight 0, its distance otherwise.
template <class Value>
LAMA_HD double tsdm_distance(const double pt[3], const TsdmParams& p, Value&& value, double grad[3])
{
    double mu[3], nu[3];
    uint32_t c[3];
    for (int k = 0; k < 3; ++k) {
        const double m = w2m_nocast(pt[k], p.scale);
        c[k] = (uint32_t)m;
        mu[k] = add_rn(m, -(double)c[k]);
        nu[k] = add_rn(1.0, -mu[k]);
    }
    if (!p.is3d) {
        const double v[4] = {value(c[0], c[1], c[2]), value(c[0] + 1, c[1], c[2]), value(c[0], c[1] + 1, c[2]), value(c[0] + 1, c[1] + 1, c[2])};
        const BeamEval e = bilinear(v, mu[0], mu[1], p.scale, 0.0, 0.0);
        grad[0] = e.gx; grad[1] = e.gy; grad[2] = 0.0;
        return e.dist;
    }
    double v[8];
    for (int i = 0; i < 8; ++i) v[i] = value(c[0] + (i & 1), c[1] + ((i >> 1) & 1), c[2] + (i >> 2));   // V000 V100 V010 V110 V001 ...
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
    grad[0] = mul_rn(-add_rn(mul_rn(a, nu[2]), mul_rn(b, mu[2])), p.scale);
    a = add_rn(mul_rn(add_rn(v[0], -v[2]), nu[0]), mul_rn(add_rn(v[1], -v[3]), mu[0]));
    b = add_rn(mul_rn(add_rn(v[4], -v[6]), nu[0]), mul_rn(add_rn(v[5], -v[7]), mu[0]));
    grad[1] = mul_rn(-add_rn(mul_rn(a, nu[2]), mul_rn(b, mu[2])), p.scale);
    a = add_rn(mul_rn(add_rn(v[0], -v[4]), nu[0]), mul_rn(add_rn(v[1], -v[5]), mu[0]));
    b = add_rn(mul_rn(add_rn(v[2], -v[6]), nu[0]), mul_rn(add_rn(v[3], -v[7]), mu[0]));
    grad[2] = mul_rn(-add_rn(mul_rn(a, nu[1]), mul_rn(b, mu[1])), p.scale);
    return dist;
}

// ---- marching cubes (toMesh :220-272) --------------------------------------------------------------------------------------
// corner i of the cube at cell c is c + (i & 1 ^ i >> 1 & 1, i >> 1 & 1, i >> 2): the reference's `delta` order
LAMA_HD void mc_corner(int i, uint32_t& dx, uint32_t& dy, uint32_t& dz)
{
    dy = (uint32_t)(i >> 1) & 1u;
    dx = ((uint32_t)i & 1u) ^ dy;
    dz = (uint32_t)i >> 2;
}
// MarchingCubes::edge_index_pairs
LAMA_HD int mc_edge_corner(int e, int end)
{
    return e < 8 ? (end ? ((e & 3) + 1) % 4 + (e & 4) : e) : (e - 8) + 4 * end;
}
// MarchingCubes::interpolate_vertex, float
LAMA_HD void mc_interpolate(const float v1[3], const float v2[3], float s1, float s2, float out[3])
{
    const float diff = fadd_rn(s1, -s2);
    if (fabs((double)diff) < 1e-6) {
        for (int k = 0; k < 3; ++k) out[k] = fmul_rn(fadd_rn(v1[k], v2[k]), 0.5f);
        return;
    }
    const float t = fdiv_rn(s1, diff);
    for (int k = 0; k < 3; ++k) out[k] = fadd_rn(v1[k], fmul_rn(t, fadd_rn(v2[k], -v1[k])));
}
// One cube of toMesh.  `cell(x, y, z, &sdf)` is get() + the weight test: false when the corner cell is absent or of weight 0.
// Returns the configuration (bit i: sdf[i] < 0), or -1 when a corner is missing; fills the corner positions and values.
template <class Cell>
LAMA_HD int mc_cube(uint32_t x, uint32_t y, uint32_t z, double scale, Cell&& cell, float pos[8][3], float sdf[8])
{
    int config = 0;
    for (int i = 0; i < 8; ++i) {
        uint32_t dx, dy, dz;
        mc_corner(i, dx, dy, dz);
        if (!cell(x + dx, y + dy, z + dz, sdf[i])) return -1;
        pos[i][0] = (float)m2w(x + dx, scale);
        pos[i][1] = (float)m2w(y + dy, scale);
        pos[i][2] = (float)m2w(z + dz, scale);
        if (sdf[i] < 0) config |= 1 << i;
    }
    return config;
}
// the vertex on crossing edge e of a cube
LAMA_HD void mc_edge_vertex(int e, const float pos[8][3], const float sdf[8], float out[3])
{
    const int a = mc_edge_corner(e, 0), b = mc_edge_corner(e, 1);
    mc_interpolate(pos[a], pos[b], sdf[a], sdf[b], out);
}

}  // namespace lama_b200
