// occ3d_oracle.cpp -- CPU restatement of the reference's 3-D occupancy maps: Map with is_3d (include/lama/sdm/map.h:125-189,
// src/sdm/map.cpp:139-157,371-455,490-529: unordered_map patches, m2p / m2c / p2m, the Container mask), FrequencyOccupancyMap
// (src/sdm/frequency_occupancy_map.cpp:38-172) and ProbabilisticOccupancyMap (src/sdm/probabilistic_occupancy_map.cpp:38-175) line
// for line, the insertion loop of GraphSlam2D::generateOccupancyMap (src/graph_slam2d.cpp:146-158) and the z-slice image of
// sdm::export_to_png (src/sdm/export.cpp:46-72), on the test oracle's w2m and Map::computeRay (oracle/lama_oracle.hpp).
// TEST INFRASTRUCTURE ONLY: compiled by tests/occ3d_oracle.py into a temporary directory, -ffp-contract=off.
#include "../../oracle/lama_oracle.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <unordered_map>
#include <vector>

using namespace orc;

namespace {

constexpr uint32_t kVolume = 32768;

struct Om {   // what the C entry points need of either map
    virtual ~Om() = default;
    virtual bool set_free(const Vec3u& c) = 0;
    virtual bool set_occupied(const Vec3u& c) = 0;
    virtual bool set_unknown(const Vec3u& c) = 0;
    virtual bool is_free(const Vec3u& c) const = 0;
    virtual bool is_occupied(const Vec3u& c) const = 0;
    virtual bool is_unknown(const Vec3u& c) const = 0;
    virtual double get_probability(const Vec3u& c) const = 0;
    virtual void prune() = 0;
    virtual bool word(const Vec3u& c, uint32_t& w) const = 0;   // the const get(): false when it returns null
    virtual int bounds(uint32_t mn[3], uint32_t mx[3]) const = 0;
    virtual bool write(const char* path) const = 0;
    virtual Vec3u w2m(const double p[3]) const = 0;
};

template <typename Cell>
struct Map3 : Om {
    SparseMap<Cell> map;   // w2m and compute_ray; its own 2-D patch table stays empty
    std::unordered_map<uint64_t, std::unique_ptr<Patch<Cell>>> patches;

    explicit Map3(double res) : map(res, 32) {}
    // map.h:153-189 with is_3d
    static uint64_t m2p(const Vec3u& c) { return ((uint64_t)(c.x >> 5) * kUniversalConstant + (c.y >> 5)) * kUniversalConstant + (c.z >> 5); }
    static uint32_t m2c(const Vec3u& c) { return (c.x & 31) | ((c.y & 31) << 5) | ((c.z & 31) << 10); }
    static Vec3u p2m(uint64_t idx)
    {
        const uint64_t uc2 = kUniversalConstant * kUniversalConstant;
        return Vec3u{(uint32_t)((idx / uc2) << 5), (uint32_t)(((idx % uc2) / kUniversalConstant) << 5), (uint32_t)(((idx % uc2) % kUniversalConstant) << 5)};
    }
    Cell* get(const Vec3u& c)   // map.cpp:371-412: allocate, set the bit
    {
        auto& p = patches[m2p(c)];
        if (!p) p.reset(new Patch<Cell>(kVolume));
        const uint32_t ci = m2c(c);
        p->set_on(ci);
        return &p->cells[ci];
    }
    const Cell* get(const Vec3u& c) const   // map.cpp:414-455, container.h:119-123
    {
        auto it = patches.find(m2p(c));
        if (it == patches.end()) return nullptr;
        const uint32_t ci = m2c(c);
        return it->second->is_on(ci) ? &it->second->cells[ci] : nullptr;
    }
    template <typename F>
    void visit_all_cells(F&& walker) const   // map.cpp:352-359
    {
        for (auto& kv : patches) {
            const Vec3u a = p2m(kv.first);
            for (uint32_t ci = 0; ci < kVolume; ++ci)
                if (kv.second->is_on(ci)) walker(Vec3u{a.x + (ci & 31), a.y + ((ci >> 5) & 31), a.z + (ci >> 10)});
        }
    }
    bool word(const Vec3u& c, uint32_t& w) const override
    {
        const Cell* cell = get(c);
        if (!cell) return false;
        std::memcpy(&w, cell, 4);
        return true;
    }
    int bounds(uint32_t mn[3], uint32_t mx[3]) const override   // map.cpp:139-157
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
    bool write(const char* path) const override   // map.cpp:490-529, container.cpp:143-176; no parameters (the occupancy maps)
    {
        FILE* f = std::fopen(path, "wb");
        if (!f) return false;
        typename SparseMap<Cell>::IOHeader h;
        std::memset(&h, 0, sizeof(h));
        h.magic = SparseMap<Cell>::kMagic; h.version = SparseMap<Cell>::kIoVersion; h.cell_size = (uint32_t)sizeof(Cell); h.patch_length = 32;
        h.num_patches = patches.size(); h.resolution = (float)map.resolution; h.is_3d = true;
        bool ok = std::fwrite(&h, sizeof(h), 1, f) == 1;
        for (auto& kv : patches) {
            ok = ok && std::fwrite(&kv.first, 8, 1, f) == 1 && std::fwrite(kv.second->cells.data(), sizeof(Cell) * kVolume, 1, f) == 1 &&
                 std::fwrite(kv.second->mask.data(), 8 * kv.second->mask.size(), 1, f) == 1;
        }
        return std::fclose(f) == 0 && ok;
    }
    Vec3u w2m(const double p[3]) const override { return map.w2m(p); }
};

class Freq3 : public Map3<FreqCell> {   // frequency_occupancy_map.cpp
public:
    using Map3<FreqCell>::Map3;
    static constexpr double occ_thresh = 0.25;   // :38
    static double prob(const FreqCell& f)        // :40-45
    {
        if (f.visited == 0) return occ_thresh;
        return ((double)f.occupied) / ((double)f.visited);
    }
    bool set_free(const Vec3u& c) override   // :65-74
    {
        FreqCell* cell = get(c);
        bool free = prob(*cell) < occ_thresh;
        cell->visited++;
        if (free) return false;
        else return (prob(*cell) < occ_thresh);
    }
    bool set_occupied(const Vec3u& c) override   // :81-91
    {
        FreqCell* cell = get(c);
        bool occupied = prob(*cell) > occ_thresh;
        cell->occupied++;
        cell->visited++;
        if (occupied) return false;
        else return (prob(*cell) > occ_thresh);
    }
    bool set_unknown(const Vec3u& c) override   // :98-108
    {
        FreqCell* cell = get(c);
        if (cell->visited == 0) return false;
        cell->occupied = 0;
        cell->visited = 0;
        return true;
    }
    bool is_free(const Vec3u& c) const override   // :115-121
    {
        const FreqCell* cell = get(c);
        if (cell == 0) return false;
        return prob(*cell) < occ_thresh;
    }
    bool is_occupied(const Vec3u& c) const override   // :128-134
    {
        const FreqCell* cell = get(c);
        if (cell == 0) return false;
        return prob(*cell) > occ_thresh;
    }
    bool is_unknown(const Vec3u& c) const override   // :141-147
    {
        const FreqCell* cell = get(c);
        if (cell == 0) return true;
        return cell->visited == 0;
    }
    void prune() override   // :149-158
    {
        visit_all_cells([&](const Vec3u& coords) {
            FreqCell* cell = const_cast<FreqCell*>(static_cast<const Freq3*>(this)->get(coords));
            if (cell->visited == 1 and (cell->occupied == 0 or cell->occupied == 1)) {
                cell->visited = 0;
                cell->occupied = 0;
            }
        });
    }
    double get_probability(const Vec3u& c) const override   // :166-172
    {
        const FreqCell* cell = get(c);
        if (cell == 0) return occ_thresh;
        return prob(*cell);
    }
};

class Prob3 : public Map3<ProbCell> {   // probabilistic_occupancy_map.cpp
public:
    static float prob(const float& logods) { return 1.0 - 1.0 / (1.0 + std::exp(logods)); }   // :38-41
    static float logods(const float& prob) { return std::log(prob / (1.0 - prob)); }         // :43-46
    double miss_, hit_, clamp_min_, clamp_max_, occ_thresh_;
    explicit Prob3(double res) : Map3<ProbCell>(res)   // :48-60
    {
        miss_ = logods(0.4);
        hit_ = logods(0.7);
        clamp_min_ = logods(0.12);
        clamp_max_ = logods(0.97);
        occ_thresh_ = 0.0 * logods(0.5);
    }
    bool set_free(const Vec3u& c) override   // :82-91
    {
        ProbCell* cell = get(c);
        bool free = cell->prob < occ_thresh_;
        cell->prob = std::max(cell->prob + miss_, clamp_min_);
        if (free) return false;
        else return (cell->prob < occ_thresh_);
    }
    bool set_occupied(const Vec3u& c) override   // :98-107
    {
        ProbCell* cell = get(c);
        bool occupied = cell->prob > occ_thresh_;
        cell->prob = std::min(cell->prob + hit_, clamp_max_);
        if (occupied) return false;
        else return (cell->prob > occ_thresh_);
    }
    bool set_unknown(const Vec3u& c) override   // :114-123
    {
        ProbCell* cell = get(c);
        bool unknown = cell->prob == occ_thresh_;
        cell->prob = occ_thresh_;
        if (unknown) return false;
        else return true;
    }
    bool is_free(const Vec3u& c) const override   // :130-136
    {
        const ProbCell* cell = get(c);
        if (cell == 0) return false;
        return cell->prob < occ_thresh_;
    }
    bool is_occupied(const Vec3u& c) const override   // :143-149
    {
        const ProbCell* cell = get(c);
        if (cell == 0) return false;
        return cell->prob > occ_thresh_;
    }
    bool is_unknown(const Vec3u& c) const override   // :156-162
    {
        const ProbCell* cell = get(c);
        if (cell == 0) return true;
        return cell->prob == occ_thresh_;
    }
    void prune() override {}
    double get_probability(const Vec3u& c) const override   // :169-175
    {
        const ProbCell* cell = get(c);
        if (cell == 0) return prob(occ_thresh_);
        return prob(cell->prob);
    }
};

}  // namespace

extern "C" {

void* o3o_create(double resolution, int kind) { return kind == 0 ? (Om*)new Freq3(resolution) : (Om*)new Prob3(resolution); }
void o3o_destroy(void* h) { delete (Om*)h; }

// generateOccupancyMap's loop (graph_slam2d.cpp:140-158) over the clouds; returns the cell updates
uint64_t o3o_insert(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, int full)
{
    Om& m = *(Om*)h;
    uint64_t cells = 0;
    for (int k = 0; k < n; ++k) {
        PointCloud pc;
        for (int i = 0; i < 3 && origins; ++i) pc.origin[i] = origins[3 * k + i];
        for (int i = 0; i < 4 && quats; ++i) pc.quat[i] = quats[4 * k + i];
        const Affine3 tf = moving_tf(pc);
        const Vec3u so = m.w2m(tf.t);
        for (int64_t i = offsets[k]; i < offsets[k + 1]; ++i) {
            double hit[3];
            tf.apply(pts + 3 * i, hit);
            m.set_occupied(m.w2m(hit));
            ++cells;
            if (full)
                SparseMap<FreqCell>::compute_ray(so, m.w2m(hit), [&](const Vec3u& coord) {
                    m.set_free(coord);
                    ++cells;
                });
        }
    }
    return cells;
}

void o3o_apply(void* h, const uint32_t* xyz, const uint8_t* ops, int n, uint8_t* changed)
{
    Om& m = *(Om*)h;
    for (int i = 0; i < n; ++i) {
        const Vec3u c{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
        const bool r = ops[i] == 0 ? m.set_free(c) : (ops[i] == 1 ? m.set_occupied(c) : m.set_unknown(c));
        if (changed) changed[i] = r;
    }
}

void o3o_query(void* h, const uint32_t* xyz, int n, double* prob, uint8_t* flags)
{
    const Om& m = *(Om*)h;
    for (int i = 0; i < n; ++i) {
        const Vec3u c{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
        prob[i] = m.get_probability(c);
        flags[i] = (uint8_t)((m.is_free(c) ? 1 : 0) | (m.is_occupied(c) ? 2 : 0) | (m.is_unknown(c) ? 4 : 0));
    }
}

void o3o_prune(void* h) { ((Om*)h)->prune(); }
int o3o_bounds(void* h, uint32_t* mn, uint32_t* mx) { return ((Om*)h)->bounds(mn, mx); }
int o3o_write(void* h, const char* path) { return ((Om*)h)->write(path) ? 1 : 0; }

void o3o_export(void* h, const uint32_t* lo, const int32_t* size, uint32_t* words, uint8_t* known)
{
    const Om& m = *(Om*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                uint32_t w = 0;
                known[i] = m.word(Vec3u{lo[0] + x, lo[1] + y, lo[2] + z}, w);
                words[i] = w;
            }
}

// build_image (export.cpp:46-72): dims = {width, height}; pixels (width per row) when out != NULL
void o3o_image(void* h, double zed, uint8_t* out, int* dims)
{
    const Om& m = *(Om*)h;
    uint32_t mn[3], mx[3];
    if (m.bounds(mn, mx) == 0) { dims[0] = dims[1] = 0; return; }
    const double zp[3] = {0, 0, zed};
    const uint32_t zmin = m.w2m(zp).z;
    dims[0] = (int)(mx[0] - mn[0]);
    dims[1] = (int)(mx[1] - mn[1]);
    if (!out) return;
    std::fill(out, out + (size_t)dims[0] * dims[1], 90);
    auto visit = [&](const Vec3u& coords) {
        if (coords.z != zmin) return;
        uint8_t& px = out[(size_t)(coords.y - mn[1]) * dims[0] + (coords.x - mn[0])];
        if (m.is_free(coords)) px = 255;
        else if (m.is_occupied(coords)) px = 0;
        else px = 127;
    };
    if (auto* f = dynamic_cast<const Freq3*>(&m)) f->visit_all_cells(visit);
    else dynamic_cast<const Prob3*>(&m)->visit_all_cells(visit);
}

}  // extern "C"
