// occ_dist3_oracle.cpp -- the reference's map update (src/slam2d.cpp:271-316, src/pf_slam2d.cpp:439-509) composed from the two CPU
// oracles, in the reference's order: for every point, setOccupied(hit) on the occupancy oracle (o3o_apply, occ3d_oracle.cpp) and, when it
// returns true, addObstacle(hit) on the distance oracle (d3o_apply, ddm3_oracle.cpp); then along Map::computeRay (the test oracle's,
// oracle/lama_oracle.hpp) setFree(c) and, when it returns true, removeObstacle(c); update() after every cloud.  Every setter call that
// returns true (an event) goes to the distance oracle: nothing is filtered.  Before each distance op its cell is read to count the ops
// that push a heap entry (an add on a cell that is not an obstacle, a remove on one that is, dynamic_distance_map.cpp:212-242); the count
// does not change what the op does.
// TEST INFRASTRUCTURE ONLY: compiled with occ3d_oracle.cpp and ddm3_oracle.cpp by tests/test_occ_dist3d.py and the check binary.
#include "../../oracle/lama_oracle.hpp"

#include <cstdint>
#include <vector>

using namespace orc;

extern "C" {
void o3o_apply(void* h, const uint32_t* xyz, const uint8_t* ops, int n, uint8_t* changed);
void d3o_apply(void* h, const uint32_t* ops, int n);
uint32_t d3o_update(void* h);
void d3o_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known);

// om: an o3o_create handle of `resolution`, dm: a d3o_create handle.  processed[k] = cloud k's update(); counts = {events, pushes}.
// Returns the cell updates.
uint64_t od3o_update_maps(void* om, void* dm, double resolution, const double* pts, const int64_t* offsets, int n, const double* origins,
                          const double* quats, int full, uint32_t* processed, uint64_t* counts)
{
    const SparseMap<FreqCell> geom(resolution, 32);   // Map::w2m of the occupancy map
    const int32_t one[3] = {1, 1, 1};
    uint64_t cells = 0, events = 0, pushes = 0;
    // one setter (op 0 setFree, 1 setOccupied); when it returns true, the distance op (kind 1 removeObstacle, 0 addObstacle)
    auto step = [&](const Vec3u& c, uint8_t op) {
        const uint32_t xyz[3] = {c.x, c.y, c.z};
        uint8_t changed = 0;
        o3o_apply(om, xyz, &op, 1, &changed);
        ++cells;
        if (!changed) return;
        const uint32_t d[4] = {c.x, c.y, c.z, op == 1 ? 0u : 1u};
        uint64_t w = 0;
        uint8_t known = 0;
        d3o_export(dm, d, one, &w, &known);
        const bool obstacle = (w >> 24 & 1u) && (w >> 32) == 0;   // valid_obstacle and sqdist 0
        ++events;
        pushes += d[3] ? obstacle : !obstacle;
        d3o_apply(dm, d, 1);
    };
    for (int k = 0; k < n; ++k) {
        PointCloud pc;
        for (int i = 0; i < 3 && origins; ++i) pc.origin[i] = origins[3 * k + i];
        for (int i = 0; i < 4 && quats; ++i) pc.quat[i] = quats[4 * k + i];
        const Affine3 tf = moving_tf(pc);
        const Vec3u so = geom.w2m(tf.t);
        for (int64_t i = offsets[k]; i < offsets[k + 1]; ++i) {
            double hit[3];
            tf.apply(pts + 3 * i, hit);
            const Vec3u mhit = geom.w2m(hit);
            step(mhit, 1);
            if (full) SparseMap<FreqCell>::compute_ray(so, mhit, [&](const Vec3u& coord) { step(coord, 0); });
        }
        processed[k] = d3o_update(dm);
    }
    counts[0] = events;
    counts[1] = pushes;
    return cells;
}

}  // extern "C"
