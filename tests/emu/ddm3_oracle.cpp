// ddm3_oracle.cpp -- CPU restatement of the reference's DynamicDistanceMap with is3d = true, line for line:
// include/lama/sdm/dynamic_distance_map.h:48-104 (distance_t, the queues), src/sdm/dynamic_distance_map.cpp:36-330 (six
// neighbours, distance, setMaxDistance, update, add/removeObstacle, raise, lower), on a 3-D Map (include/lama/sdm/map.h:125-189,
// src/sdm/map.cpp:139-157,371-455,490-529: unordered_map patches of 32^3 cells with the Container mask, the mutable and const get,
// bounds, write), the same 3-D Map restatement as occ3d_oracle.cpp, and the z-slice image of sdm::export_to_png
// (src/sdm/export.cpp:74-96).  Uses the test oracle's w2m (oracle/lama_oracle.hpp).
// TEST INFRASTRUCTURE ONLY: compiled by tests/ddm3_oracle.py into a temporary directory, -ffp-contract=off.
#include "../../oracle/lama_oracle.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <queue>
#include <unordered_map>
#include <vector>

using namespace orc;

namespace {

constexpr uint32_t kVolume = 32768;

struct distance_t {   // dynamic_distance_map.h:48-53, 10 bytes
    int16_t obstacle[3];
    uint16_t sqdist;
    bool valid_obstacle;
    bool is_queued;
};
static_assert(sizeof(distance_t) == 10, "distance_t");

struct Map3 {
    SparseMap<distance_t> map;   // w2m; its own 2-D patch table stays empty
    std::unordered_map<uint64_t, std::unique_ptr<Patch<distance_t>>> patches;

    explicit Map3(double res) : map(res, 32) {}
    static uint64_t m2p(const Vec3u& c) { return ((uint64_t)(c.x >> 5) * kUniversalConstant + (c.y >> 5)) * kUniversalConstant + (c.z >> 5); }
    static uint32_t m2c(const Vec3u& c) { return (c.x & 31) | ((c.y & 31) << 5) | ((c.z & 31) << 10); }
    static Vec3u p2m(uint64_t idx)
    {
        const uint64_t uc2 = kUniversalConstant * kUniversalConstant;
        return Vec3u{(uint32_t)((idx / uc2) << 5), (uint32_t)(((idx % uc2) / kUniversalConstant) << 5), (uint32_t)(((idx % uc2) % kUniversalConstant) << 5)};
    }
    distance_t* get(const Vec3u& c)   // map.cpp:371-412
    {
        auto& p = patches[m2p(c)];
        if (!p) p.reset(new Patch<distance_t>(kVolume));
        const uint32_t ci = m2c(c);
        p->set_on(ci);
        return &p->cells[ci];
    }
    const distance_t* get(const Vec3u& c) const   // map.cpp:414-455
    {
        auto it = patches.find(m2p(c));
        if (it == patches.end()) return nullptr;
        const uint32_t ci = m2c(c);
        return it->second->is_on(ci) ? &it->second->cells[ci] : nullptr;
    }
    int bounds(uint32_t mn[3], uint32_t mx[3]) const   // map.cpp:139-157
    {
        for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
        for (auto& kv : patches) {
            const Vec3u a = p2m(kv.first);
            const uint32_t v[3] = {a.x, a.y, a.z};
            for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], v[k]); mx[k] = std::max(mx[k], v[k]); }
        }
        for (int k = 0; k < 3; ++k) mx[k] += 32;
        return (int)patches.size();
    }
};

class Ddm3 : public Map3 {
public:
    typedef std::pair<int, Vec3u> queue_pair_t;
    struct compare_prio {
        bool operator()(const queue_pair_t& left, const queue_pair_t& right) const { return left.first > right.first; }
    };
    typedef std::priority_queue<queue_pair_t, std::vector<queue_pair_t>, compare_prio> queue_t;
    queue_t lower_, raise_;
    int deltas_[6][3] = {{1, 0, 0}, {0, 1, 0}, {-1, 0, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};   // :40-45
    uint32_t max_sqdist_ = 100;                                                                   // :38

    explicit Ddm3(double res) : Map3(res) {}

    static Vec3u add(const Vec3u& a, int64_t dx, int64_t dy, int64_t dz)   // (a.cast<int64_t>() + d).cast<uint32_t>()
    {
        return Vec3u{(uint32_t)((int64_t)a.x + dx), (uint32_t)((int64_t)a.y + dy), (uint32_t)((int64_t)a.z + dz)};
    }

    double distance(const Vec3u& c) const   // :140-147
    {
        const distance_t* cell = get(c);
        if (cell == 0 || not cell->valid_obstacle) return std::sqrt((double)max_sqdist_) * map.resolution;
        return std::sqrt((double)cell->sqdist) * map.resolution;
    }
    double distance(const double p[3], double* gradient) const   // :66-138, is_3d branch
    {
        double m[3];
        map.w2m_nocast(p, m);
        const Vec3u d{(uint32_t)m[0], (uint32_t)m[1], (uint32_t)m[2]};
        const double mu[3] = {m[0] - (double)d.x, m[1] - (double)d.y, m[2] - (double)d.z};
        const double muinv[3] = {1.0 - mu[0], 1.0 - mu[1], 1.0 - mu[2]};
        double val[8];
        val[0] = distance(d);
        val[1] = distance(Vec3u{d.x + 1, d.y, d.z});
        val[2] = distance(Vec3u{d.x, d.y + 1, d.z});
        val[3] = distance(Vec3u{d.x + 1, d.y + 1, d.z});
        val[4] = distance(Vec3u{d.x, d.y, d.z + 1});
        val[5] = distance(Vec3u{d.x + 1, d.y, d.z + 1});
        val[6] = distance(Vec3u{d.x, d.y + 1, d.z + 1});
        val[7] = distance(Vec3u{d.x + 1, d.y + 1, d.z + 1});
        const double dist = val[0] * (muinv[0] * muinv[1] * muinv[2]) +
                            val[1] * mu[0] * muinv[1] * muinv[2] +
                            val[2] * muinv[0] * mu[1] * muinv[2] +
                            val[3] * mu[0] * mu[1] * muinv[2] +
                            val[4] * muinv[0] * muinv[1] * mu[2] +
                            val[5] * mu[0] * muinv[1] * mu[2] +
                            val[6] * muinv[0] * mu[1] * mu[2] +
                            val[7] * (mu[0] * mu[1] * mu[2]);
        if (gradient) {
            const double scale = map.scale;
            double a, b;
            a = (val[0] - val[1]) * muinv[1] + (val[2] - val[3]) * mu[1];
            b = (val[4] - val[5]) * muinv[1] + (val[6] - val[7]) * mu[1];
            gradient[0] = -(a * muinv[2] + b * mu[2]) * scale;
            a = (val[0] - val[2]) * muinv[0] + (val[1] - val[3]) * mu[0];
            b = (val[4] - val[6]) * muinv[0] + (val[5] - val[7]) * mu[0];
            gradient[1] = -(a * muinv[2] + b * mu[2]) * scale;
            a = (val[0] - val[4]) * muinv[0] + (val[1] - val[5]) * mu[0];
            b = (val[2] - val[6]) * muinv[0] + (val[3] - val[7]) * mu[0];
            gradient[2] = -(a * muinv[1] + b * mu[1]) * scale;
        }
        return dist;
    }
    void setMaxDistance(double distance)   // :149-153
    {
        max_sqdist_ = std::ceil(distance * map.scale);
        max_sqdist_ *= max_sqdist_;
    }
    double maxDistance() const { return std::sqrt((double)(max_sqdist_)) * map.resolution; }   // :155-158

    uint32_t update()   // :160-197
    {
        uint32_t number_of_proccessed_cells = 0;
        while (not raise_.empty()) {
            Vec3u location = raise_.top().second; raise_.pop();
            distance_t* current = get(location);
            if (current == 0) continue;
            ++number_of_proccessed_cells;
            raise(location, *current);
        }
        while (not lower_.empty()) {
            Vec3u location = lower_.top().second; lower_.pop();
            distance_t* current = get(location);
            ++number_of_proccessed_cells;
            if (current == 0) continue;
            if (current->valid_obstacle) {
                Vec3u obs = add(location, current->obstacle[0], current->obstacle[1], current->obstacle[2]);
                const distance_t* obstacle = get(obs);
                if (obstacle == 0) continue;
                if (obstacle->sqdist == 0) lower(location, *current);
            }
        }
        return number_of_proccessed_cells;
    }
    void addObstacle(const Vec3u& location)   // :212-226
    {
        distance_t* cell = get(location);
        if (cell == nullptr) return;
        if ((cell->valid_obstacle and cell->sqdist == 0)) return;
        cell->sqdist = 0;
        cell->obstacle[0] = cell->obstacle[1] = cell->obstacle[2] = 0;
        cell->valid_obstacle = true;
        cell->is_queued = true;
        lower_.push({0, location});
    }
    void removeObstacle(const Vec3u& location)   // :228-242
    {
        distance_t* cell = get(location);
        if (cell == nullptr) return;
        if (not(cell->valid_obstacle and cell->sqdist == 0)) return;
        cell->sqdist = 0;
        cell->obstacle[0] = cell->obstacle[1] = cell->obstacle[2] = 0;
        cell->valid_obstacle = false;
        cell->is_queued = true;
        raise_.push({0, location});
    }
    void raise(const Vec3u& location, distance_t& current)   // :244-279
    {
        for (int i = 0; i < 6; ++i) {
            const Vec3u newloc = add(location, deltas_[i][0], deltas_[i][1], deltas_[i][2]);
            distance_t* neighbor = get(newloc);
            if (neighbor->is_queued or (not neighbor->valid_obstacle)) continue;
            const Vec3u obs = add(newloc, neighbor->obstacle[0], neighbor->obstacle[1], neighbor->obstacle[2]);
            const distance_t* obstacle = get(obs);
            if (obstacle == 0) continue;
            if (not(obstacle->valid_obstacle)) {
                raise_.push({neighbor->sqdist, newloc});
                neighbor->sqdist = 0;
                neighbor->obstacle[0] = neighbor->obstacle[1] = neighbor->obstacle[2] = 0;
                neighbor->valid_obstacle = false;
                neighbor->is_queued = true;
            } else if (not neighbor->is_queued) {
                lower_.push({neighbor->sqdist, newloc});
                neighbor->is_queued = true;
            }
        }
        current.is_queued = false;
    }
    void lower(const Vec3u& location, distance_t& current)   // :281-330
    {
        if (not current.is_queued) return;
        for (int i = 0; i < 6; ++i) {
            const int64_t d[3] = {deltas_[i][0], deltas_[i][1], deltas_[i][2]};
            if (d[0] * current.obstacle[0] > 0 || d[1] * current.obstacle[1] > 0 || d[2] * current.obstacle[2] > 0) continue;
            const int64_t newloc[3] = {(int64_t)location.x + d[0], (int64_t)location.y + d[1], (int64_t)location.z + d[2]};
            const Vec3u nl{(uint32_t)newloc[0], (uint32_t)newloc[1], (uint32_t)newloc[2]};
            distance_t* neighbor = get(nl);
            const int64_t obs[3] = {(int64_t)location.x + current.obstacle[0], (int64_t)location.y + current.obstacle[1],
                                    (int64_t)location.z + current.obstacle[2]};
            const int64_t dist[3] = {newloc[0] - obs[0], newloc[1] - obs[1], newloc[2] - obs[2]};
            uint32_t new_sqdist = dist[0] * dist[0] + dist[1] * dist[1] + dist[2] * dist[2];
            uint32_t cmp_sqdist = neighbor->valid_obstacle ? neighbor->sqdist : max_sqdist_;
            bool overwrite = (new_sqdist < cmp_sqdist);
            if (not overwrite && new_sqdist == neighbor->sqdist) {
                const Vec3u nobs = add(nl, neighbor->obstacle[0], neighbor->obstacle[1], neighbor->obstacle[2]);
                const distance_t* obstacle = get(nobs);
                if (not neighbor->valid_obstacle || (obstacle != 0 && not(obstacle->valid_obstacle and obstacle->sqdist == 0))) overwrite = true;
            }
            if (overwrite) {
                lower_.push({(int)new_sqdist, nl});
                neighbor->sqdist = new_sqdist;
                neighbor->valid_obstacle = true;
                for (int k = 0; k < 3; ++k) neighbor->obstacle[k] = (int16_t)(obs[k] - newloc[k]);
                neighbor->is_queued = true;
            }
        }
        current.is_queued = false;
    }

    bool write(const char* path) const   // map.cpp:490-529 with is_3d, then writeParameters (:200-203)
    {
        FILE* f = std::fopen(path, "wb");
        if (!f) return false;
        SparseMap<distance_t>::IOHeader h;
        std::memset(&h, 0, sizeof(h));
        h.magic = SparseMap<distance_t>::kMagic; h.version = SparseMap<distance_t>::kIoVersion; h.cell_size = (uint32_t)sizeof(distance_t);
        h.patch_length = 32; h.num_patches = patches.size(); h.resolution = (float)map.resolution; h.is_3d = true;
        bool ok = std::fwrite(&h, sizeof(h), 1, f) == 1 && std::fwrite(&max_sqdist_, 4, 1, f) == 1;
        for (auto& kv : patches)
            ok = ok && std::fwrite(&kv.first, 8, 1, f) == 1 && std::fwrite(kv.second->cells.data(), sizeof(distance_t) * kVolume, 1, f) == 1 &&
                 std::fwrite(kv.second->mask.data(), 8 * kv.second->mask.size(), 1, f) == 1;
        return std::fclose(f) == 0 && ok;
    }
};

}  // namespace

extern "C" {

void* d3o_create(double resolution, double l2_max)
{
    Ddm3* m = new Ddm3(resolution);
    m->setMaxDistance(l2_max);
    return m;
}
void d3o_destroy(void* h) { delete (Ddm3*)h; }
uint32_t d3o_max_sqdist(void* h) { return ((Ddm3*)h)->max_sqdist_; }
double d3o_max_distance(void* h) { return ((Ddm3*)h)->maxDistance(); }

// ops: x, y, z, kind (0 addObstacle, 1 removeObstacle) per op, applied in list order
void d3o_apply(void* h, const uint32_t* ops, int n)
{
    Ddm3& m = *(Ddm3*)h;
    for (int i = 0; i < n; ++i) {
        const Vec3u c{ops[4 * i], ops[4 * i + 1], ops[4 * i + 2]};
        if (ops[4 * i + 3]) m.removeObstacle(c);
        else m.addObstacle(c);
    }
}
uint32_t d3o_update(void* h) { return ((Ddm3*)h)->update(); }

void d3o_distance(void* h, const double* pts, int n, double* dist, double* grad)
{
    const Ddm3& m = *(Ddm3*)h;
    for (int i = 0; i < n; ++i) dist[i] = m.distance(pts + 3 * i, grad ? grad + 3 * i : nullptr);
}
void d3o_cell_distance(void* h, const uint32_t* xyz, int n, double* dist)
{
    const Ddm3& m = *(Ddm3*)h;
    for (int i = 0; i < n; ++i) dist[i] = m.distance(Vec3u{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
}
int d3o_bounds(void* h, uint32_t* mn, uint32_t* mx) { return ((Ddm3*)h)->bounds(mn, mx); }
// the patch ids (Map::m2p), any order
int d3o_patch_ids(void* h, uint64_t* ids)
{
    const Ddm3& m = *(Ddm3*)h;
    int i = 0;
    for (auto& kv : m.patches) ids[i++] = kv.first;
    return i;
}
// the box lo + [0, size), x fastest: cells as the device word (ddm3_core.h layout) and known bits; an absent patch reads 0
void d3o_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known)
{
    const Ddm3& m = *(Ddm3*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                const Vec3u c{lo[0] + x, lo[1] + y, lo[2] + z};
                auto it = m.patches.find(Map3::m2p(c));
                uint64_t w = 0;
                uint8_t k = 0;
                if (it != m.patches.end()) {
                    const uint32_t ci = Map3::m2c(c);
                    const distance_t& d = it->second->cells[ci];
                    k = it->second->is_on(ci);
                    w = (uint64_t)(uint8_t)d.obstacle[0] | ((uint64_t)(uint8_t)d.obstacle[1] << 8) | ((uint64_t)(uint8_t)d.obstacle[2] << 16) |
                        ((uint64_t)((d.valid_obstacle ? 1u : 0u) | (d.is_queued ? 2u : 0u) | (k ? 4u : 0u)) << 24) | ((uint64_t)d.sqdist << 32);
                }
                words[i] = w;
                known[i] = k;
            }
}
int d3o_write(void* h, const char* path) { return ((Ddm3*)h)->write(path) ? 1 : 0; }

// build_image (export.cpp:74-96): dims = {width, height}; pixels (width per row) when out != NULL
void d3o_image(void* h, double zed, uint8_t* out, int* dims)
{
    const Ddm3& m = *(Ddm3*)h;
    uint32_t mn[3], mx[3];
    if (m.bounds(mn, mx) == 0) { dims[0] = dims[1] = 0; return; }
    const double zp[3] = {0, 0, zed};
    const uint32_t zmin = m.map.w2m(zp).z;
    dims[0] = (int)(mx[0] - mn[0]);
    dims[1] = (int)(mx[1] - mn[1]);
    if (!out) return;
    std::fill(out, out + (size_t)dims[0] * dims[1], 127);
    for (auto& kv : m.patches) {   // visit_all_cells (map.cpp:352-359)
        const Vec3u a = Map3::p2m(kv.first);
        for (uint32_t ci = 0; ci < kVolume; ++ci) {
            if (!kv.second->is_on(ci)) continue;
            const Vec3u c{a.x + (ci & 31), a.y + ((ci >> 5) & 31), a.z + (ci >> 10)};
            if (c.z != zmin) continue;
            out[(size_t)(c.y - mn[1]) * dims[0] + (c.x - mn[0])] = (uint8_t)(m.distance(c) * 255 / m.maxDistance());
        }
    }
}

}  // extern "C"
