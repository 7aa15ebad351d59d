// global_map_oracle.cpp -- CPU restatement of GraphSlam2D::generateOccupancyMap's loop (src/graph_slam2d.cpp:131-164) and of
// FrequencyOccupancyMap::prune (src/sdm/frequency_occupancy_map.cpp:149-158) on the test oracle's map (oracle/lama_oracle.hpp).
// TEST INFRASTRUCTURE ONLY: compiled by tests/global_map_oracle.py into a temporary directory.
#include "../../oracle/lama_oracle.hpp"

#include <cmath>

using namespace orc;

namespace {

// FrequencyOccupancyMap::prune: every known cell visited once and occupied at most once goes back to {0, 0}; its known bit stays
// (the mutable get() that reads it sets the bit, which is on already)
void prune(FrequencyOccupancyMap& occ)
{
    occ.visit_all_cells([&](const Vec3u& c) {
        FreqCell* cell = occ.get(c);
        if (cell->visited == 1 && (cell->occupied == 0 || cell->occupied == 1)) {
            cell->visited  = 0;
            cell->occupied = 0;
        }
    });
}

}  // namespace

extern "C" {

void* gmo_create(double resolution, uint32_t patch) { return new FrequencyOccupancyMap(resolution, patch); }
void gmo_destroy(void* m) { delete (FrequencyOccupancyMap*)m; }

// graph_slam2d.cpp:135-160 for scans k = points [offsets[k], offsets[k + 1]) at SE2 states + 4k = {cos, sin, x, y}; thetas (may be
// null) overrides pose.rotation() = atan2(sin, cos) per scan, for poses known as (x, y, theta) only
uint64_t gmo_insert_scans(void* m, const double* pts, const int64_t* offsets, int n_scans, const double* origins, const double* quats, const double* states,
                          const double* thetas, int full)
{
    auto& occ = *(FrequencyOccupancyMap*)m;
    uint64_t cells = 0;
    for (int k = 0; k < n_scans; ++k) {
        PointCloud pc;
        for (int i = 0; i < 3; ++i) pc.origin[i] = origins ? origins[3 * k + i] : 0.0;
        for (int i = 0; i < 4; ++i) pc.quat[i] = quats ? quats[4 * k + i] : (i == 3 ? 1.0 : 0.0);
        // Isometry3d moving_tf = Translation3d(sensor_origin) * sensor_orientation;
        // Isometry3d fixed_tf  = Translation3d(pose.x(), pose.y(), 0.0) * AngleAxisd(pose.rotation(), UnitZ);  tf = fixed_tf * moving_tf
        const double* s = states + 4 * k;
        const Affine3 tf = compose(fixed_tf(s[2], s[3], thetas ? thetas[k] : std::atan2(s[1], s[0])), moving_tf(pc));
        const double origin[3] = {tf.t[0], tf.t[1], tf.t[2]};
        const Vec3u so = occ.w2m(origin);
        for (int64_t b = offsets[k]; b < offsets[k + 1]; ++b) {
            double hit[3];
            tf.apply(pts + 3 * b, hit);
            const Vec3u h = occ.w2m(hit);
            occ.set_occupied(h);
            ++cells;
            if (full)
                FrequencyOccupancyMap::compute_ray(so, h, [&](const Vec3u& c) {
                    occ.set_free(c);
                    ++cells;
                });
        }
    }
    return cells;
}

void gmo_prune(void* m) { prune(*(FrequencyOccupancyMap*)m); }

int gmo_bounds(void* m, uint32_t* mn, uint32_t* mx)
{
    Vec3u a, b;
    auto& occ = *(FrequencyOccupancyMap*)m;
    if (!occ.bounds(a, b)) return 0;
    mn[0] = a.x; mn[1] = a.y; mx[0] = b.x; mx[1] = b.y;
    return (int)occ.num_patches();
}

// the patch keys (Map::m2p) of the map, in no particular order; returns their number
int gmo_patches(void* m, uint64_t* keys, int cap)
{
    auto& occ = *(FrequencyOccupancyMap*)m;
    int i = 0;
    for (auto& kv : occ.patches)
        if (i < cap) keys[i++] = kv.first;
    return (int)occ.patches.size();
}

void gmo_export(void* m, uint32_t x0, uint32_t y0, int w, int h, uint16_t* occupied, uint16_t* visited, uint8_t* known)
{
    const auto& occ = *(const FrequencyOccupancyMap*)m;
    for (int j = 0; j < h; ++j)
        for (int i = 0; i < w; ++i) {
            const FreqCell* c = occ.get(Vec3u{x0 + (uint32_t)i, y0 + (uint32_t)j, 0});
            const size_t k = (size_t)j * w + i;
            occupied[k] = c ? c->occupied : 0;
            visited[k]  = c ? c->visited : 0;
            known[k]    = c ? 1 : 0;
        }
}

// getProbability / isFree / isOccupied / isUnknown: flags bit 0 free, bit 1 occupied, bit 2 unknown
void gmo_query(void* m, const uint32_t* cells, int n, double* prob, uint8_t* flags)
{
    const auto& occ = *(const FrequencyOccupancyMap*)m;
    for (int i = 0; i < n; ++i) {
        const Vec3u c{cells[2 * i], cells[2 * i + 1], 0};
        prob[i]  = occ.get_probability(c);
        flags[i] = (uint8_t)((occ.is_free(c) ? 1 : 0) | (occ.is_occupied(c) ? 2 : 0) | (occ.is_unknown(c) ? 4 : 0));
    }
}

int gmo_write(void* m, const char* path) { return ((FrequencyOccupancyMap*)m)->write(path, nullptr, 0) ? 1 : 0; }

int gmo_image(void* m, uint8_t* out, size_t cap, int* dims)
{
    uint32_t w, h;
    const auto img = occupancy_image(*(const FrequencyOccupancyMap*)m, w, h);
    dims[0] = (int)w; dims[1] = (int)h;
    if (out && cap >= img.size()) std::memcpy(out, img.data(), img.size());
    return 1;
}

}  // extern "C"
