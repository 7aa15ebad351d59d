// tsdm_oracle.cpp -- CPU restatement of lama::TruncatedSignedDistanceMap (src/sdm/truncated_signed_distance_map.cpp), of
// MarchingCubes' vertex interpolation (src/sdm/marching_cubes.cpp) and of sdm::export_to_ply (src/sdm/export.cpp:112-143), on the
// test oracle's addressing and Map::computeRay (oracle/lama_oracle.hpp), with 3-D m2p / m2c / p2m added.  toMesh uses the
// product's generated triangle table (iris_lama_b200/csrc/mc_table.h) and visits patches in ascending (z, y, x) anchor order, then
// cell index: the order the device defines where the reference iterates an unordered_map.
// TEST INFRASTRUCTURE ONLY: compiled by tests/tsdm_oracle.py into a temporary directory, -ffp-contract=off.
#include "../../oracle/lama_oracle.hpp"
#include "../../iris_lama_b200/csrc/mc_table.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <unordered_map>
#include <unordered_set>
#include <vector>

using namespace orc;
using lama_b200::kMcRow;
using lama_b200::McTable;
using lama_b200::mc_build_table;

namespace {

struct Tsd {   // tsd_t, truncated_signed_distance_map.h:43-46
    float distance;
    float weight;
};

struct KeyHash {   // types.h KeyHash
    size_t operator()(const Vec3u& k) const { return k.z + 2642244ul * (k.y + k.x * 2642244ul); }
};

template <typename T> int sign(T val) { return (T(0) < val) - (val < T(0)); }   // types.h:101-103

struct Tsdm {
    SparseMap<Tsd> map;   // w2m / m2w / compute_ray; its own 2-D patch table stays empty
    bool is3d;
    uint32_t volume;
    std::unordered_map<uint64_t, std::unique_ptr<Patch<Tsd>>> patches;
    float maximum_weight = 10000, truncate_size = 0.15f, epsilon, delta;

    Tsdm(double res, bool three_d) : map(res, 32), is3d(three_d), volume(three_d ? 32768u : 1024u)
    {
        epsilon = (float)res;
        delta = (float)(4 * res);
    }
    // map.h:153-189 with is_3d
    uint64_t m2p(const Vec3u& c) const
    {
        if (is3d) return ((uint64_t)(c.x >> 5) * kUniversalConstant + (c.y >> 5)) * kUniversalConstant + (c.z >> 5);
        return (uint64_t)(c.x >> 5) * kUniversalConstant + (c.y >> 5);
    }
    uint32_t m2c(const Vec3u& c) const { return (c.x & 31) | ((c.y & 31) << 5) | (is3d ? (c.z & 31) << 10 : 0u); }
    Vec3u p2m(uint64_t idx) const
    {
        if (is3d) {
            const uint64_t uc2 = kUniversalConstant * kUniversalConstant;
            return Vec3u{(uint32_t)((idx / uc2) << 5), (uint32_t)(((idx % uc2) / kUniversalConstant) << 5), (uint32_t)(((idx % uc2) % kUniversalConstant) << 5)};
        }
        return Vec3u{(uint32_t)((idx / kUniversalConstant) << 5), (uint32_t)((idx % kUniversalConstant) << 5), 0};
    }
    Tsd* get_mut(const Vec3u& c)   // map.cpp:371-412: allocate, set the bit
    {
        auto& p = patches[m2p(c)];
        if (!p) p.reset(new Patch<Tsd>(volume));
        const uint32_t ci = m2c(c);
        p->set_on(ci);
        return &p->cells[ci];
    }
    const Tsd* get(const Vec3u& c) const   // map.cpp:414-455
    {
        auto it = patches.find(m2p(c));
        if (it == patches.end()) return nullptr;
        const uint32_t ci = m2c(c);
        return it->second->is_on(ci) ? &it->second->cells[ci] : nullptr;
    }
    double distance_cell(const Vec3u& c) const   // :132-139
    {
        const Tsd* cell = get(c);
        if (cell == nullptr || cell->weight == 0.0) return truncate_size;
        return cell->distance;
    }

    void integrate(const double origin[3], const double hit[3])   // :161-208
    {
        double dir[3];
        for (int k = 0; k < 3; ++k) dir[k] = hit[k] - origin[k];
        const double sq = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
        float squared_norm = sq;
        if (sq > 0) {
            const double n = std::sqrt(sq);
            for (int k = 0; k < 3; ++k) dir[k] /= n;
        }
        float truncate = std::min(squared_norm, truncate_size);
        double s[3], e[3];
        for (int k = 0; k < 3; ++k) {
            s[k] = hit[k] - dir[k] * (double)truncate;
            e[k] = hit[k] + dir[k] * (double)truncate_size;
        }
        const float inv_squared_norm = 1.0 / squared_norm;
        const float inv_delta_less_epsilon = 1.0 / (delta - epsilon);
        SparseMap<Tsd>::compute_ray(map.w2m(s), map.w2m(e), [&](const Vec3u& c) {
            Tsd* cell = get_mut(c);
            double vc[3], oh[3], ch[3];
            map.m2w(c, vc);
            for (int k = 0; k < 3; ++k) {
                oh[k] = hit[k] - origin[k];
                ch[k] = hit[k] - vc[k];
            }
            float distance = std::sqrt((ch[0] * ch[0] + ch[1] * ch[1]) + ch[2] * ch[2]) * sign((ch[0] * oh[0] + ch[1] * oh[1]) + ch[2] * oh[2]);
            float weight;
            if (distance < -delta) return;
            else if (-delta <= distance && distance <= -epsilon) weight = (distance + delta) * inv_squared_norm * inv_delta_less_epsilon;
            else weight = inv_squared_norm;
            cell->distance = (cell->weight * cell->distance + weight * distance) / (cell->weight + weight);
            cell->weight = std::min(cell->weight + weight, maximum_weight);
        });
    }

    size_t insert(const PointCloud& pc)   // :141-158
    {
        const Affine3 a = moving_tf(pc);
        std::unordered_set<Vec3u, KeyHash> keys;
        for (size_t i = 0; i < pc.size(); ++i) {
            double hit[3];
            a.apply(&pc.pts[3 * i], hit);
            if (!keys.insert(map.w2m(hit)).second) continue;
            integrate(pc.origin, hit);
        }
        return keys.size();
    }

    double distance(const double p[3], double grad[3]) const   // :59-130
    {
        double m[3], mu[3], muinv[3];
        uint32_t dc[3];
        map.w2m_nocast(p, m);
        for (int k = 0; k < 3; ++k) {
            dc[k] = (uint32_t)m[k];
            mu[k] = m[k] - (double)dc[k];
            muinv[k] = 1.0 - mu[k];
        }
        auto val = [&](uint32_t dx, uint32_t dy, uint32_t dz) { return distance_cell(Vec3u{dc[0] + dx, dc[1] + dy, dc[2] + dz}); };
        if (!is3d) {
            const double v0 = val(0, 0, 0), v1 = val(1, 0, 0), v2 = val(0, 1, 0), v3 = val(1, 1, 0);
            const double dist = v0 * muinv[0] * muinv[1] + v1 * muinv[1] * mu[0] + v2 * muinv[0] * mu[1] + v3 * mu[0] * mu[1];
            grad[0] = -((v0 - v1) * muinv[1] + (v2 - v3) * mu[1]) * map.scale;
            grad[1] = -((v0 - v2) * muinv[0] + (v1 - v3) * mu[0]) * map.scale;
            grad[2] = 0;
            return dist;
        }
        const double v[8] = {val(0, 0, 0), val(1, 0, 0), val(0, 1, 0), val(1, 1, 0), val(0, 0, 1), val(1, 0, 1), val(0, 1, 1), val(1, 1, 1)};
        const double dist = v[0] * ((muinv[0] * muinv[1]) * muinv[2]) + v[1] * mu[0] * muinv[1] * muinv[2] + v[2] * muinv[0] * mu[1] * muinv[2] +
                            v[3] * mu[0] * mu[1] * muinv[2] + v[4] * muinv[0] * muinv[1] * mu[2] + v[5] * mu[0] * muinv[1] * mu[2] +
                            v[6] * muinv[0] * mu[1] * mu[2] + v[7] * ((mu[0] * mu[1]) * mu[2]);
        double a, b;
        a = (v[0] - v[1]) * muinv[1] + (v[2] - v[3]) * mu[1];
        b = (v[4] - v[5]) * muinv[1] + (v[6] - v[7]) * mu[1];
        grad[0] = -(a * muinv[2] + b * mu[2]) * map.scale;
        a = (v[0] - v[2]) * muinv[0] + (v[1] - v[3]) * mu[0];
        b = (v[4] - v[6]) * muinv[0] + (v[5] - v[7]) * mu[0];
        grad[1] = -(a * muinv[2] + b * mu[2]) * map.scale;
        a = (v[0] - v[4]) * muinv[0] + (v[1] - v[5]) * mu[0];
        b = (v[2] - v[6]) * muinv[0] + (v[3] - v[7]) * mu[0];
        grad[2] = -(a * muinv[1] + b * mu[1]) * map.scale;
        return dist;
    }

    std::vector<uint64_t> ordered_patches() const   // ascending (z, y, x) anchor
    {
        std::vector<uint64_t> keys;
        for (auto& kv : patches) keys.push_back(kv.first);
        std::sort(keys.begin(), keys.end(), [&](uint64_t a, uint64_t b) {
            const Vec3u pa = p2m(a), pb = p2m(b);
            if (pa.z != pb.z) return pa.z < pb.z;
            if (pa.y != pb.y) return pa.y < pb.y;
            return pa.x < pb.x;
        });
        return keys;
    }

    void to_mesh(std::vector<float>& out) const   // :220-272
    {
        static const McTable table = mc_build_table();
        static const uint32_t delta_[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
        static const int edge_pairs[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6}, {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
        for (uint64_t key : ordered_patches()) {
            const Vec3u a = p2m(key);
            const Patch<Tsd>& p = *patches.at(key);
            for (uint32_t ci = 0; ci < volume; ++ci) {
                if (!p.is_on(ci)) continue;
                const Vec3u c{a.x + (ci & 31), a.y + ((ci >> 5) & 31), is3d ? a.z + (ci >> 10) : 0u};
                float vtx[8][3], sdf[8];
                bool valid = true;
                for (int i = 0; i < 8 && valid; ++i) {
                    const Vec3u q{c.x + delta_[i][0], c.y + delta_[i][1], c.z + delta_[i][2]};
                    const Tsd* cell = get(q);
                    if (cell == nullptr || cell->weight == 0.0) { valid = false; break; }
                    double w[3];
                    map.m2w(q, w);
                    for (int k = 0; k < 3; ++k) vtx[i][k] = (float)w[k];
                    sdf[i] = (float)distance_cell(q);
                }
                if (!valid) continue;
                int config = 0;
                for (int i = 0; i < 8; ++i) config |= sdf[i] < 0 ? (1 << i) : 0;
                float edge[12][3];
                for (int e = 0; e < 12; ++e) {   // interpolate_edge_vertices, interpolate_vertex
                    const int e0 = edge_pairs[e][0], e1 = edge_pairs[e][1];
                    if (!((sdf[e0] < 0.0f && sdf[e1] >= 0.0f) || (sdf[e0] >= 0.0f && sdf[e1] < 0.0f))) continue;
                    const float diff = sdf[e0] - sdf[e1];
                    if (std::fabs(diff) < 1e-6) {
                        for (int k = 0; k < 3; ++k) edge[e][k] = (vtx[e0][k] + vtx[e1][k]) * 0.5f;
                    } else {
                        const float t = sdf[e0] / diff;
                        for (int k = 0; k < 3; ++k) edge[e][k] = vtx[e0][k] + t * (vtx[e1][k] - vtx[e0][k]);
                    }
                }
                for (int j = 0; table.tri[config][j] != -1; ++j)
                    for (int k = 0; k < 3; ++k) out.push_back(edge[table.tri[config][j]][k]);
            }
        }
    }
};

}  // namespace

extern "C" {

void* tso_create(double resolution, int is3d) { return new Tsdm(resolution, is3d != 0); }
void tso_destroy(void* h) { delete (Tsdm*)h; }
void tso_set_max_distance(void* h, double d) { ((Tsdm*)h)->truncate_size = (float)d; }

void tso_insert(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, uint64_t* out)
{
    for (int k = 0; k < n; ++k) {
        PointCloud pc;
        pc.pts.assign(pts + 3 * offsets[k], pts + 3 * offsets[k + 1]);
        for (int i = 0; i < 3 && origins; ++i) pc.origin[i] = origins[3 * k + i];
        for (int i = 0; i < 4 && quats; ++i) pc.quat[i] = quats[4 * k + i];
        const size_t r = ((Tsdm*)h)->insert(pc);
        if (out) out[k] = r;
    }
}

void tso_integrate(void* h, const double* origin, const double* hit) { ((Tsdm*)h)->integrate(origin, hit); }

void tso_distance(void* h, const double* pts, int n, double* dist, double* grad)
{
    for (int i = 0; i < n; ++i) dist[i] = ((Tsdm*)h)->distance(pts + 3 * i, grad + 3 * i);
}

int tso_bounds(void* h, uint32_t* mn, uint32_t* mx)   // Map::bounds (map.cpp:139-157)
{
    const Tsdm& t = *(Tsdm*)h;
    for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
    for (auto& kv : t.patches) {
        const Vec3u a = t.p2m(kv.first);
        const uint32_t v[3] = {a.x, a.y, a.z};
        for (int k = 0; k < 3; ++k) { mn[k] = std::min(mn[k], v[k]); mx[k] = std::max(mx[k], v[k]); }
    }
    for (int k = 0; k < 3; ++k) mx[k] += 32;
    return (int)t.patches.size();
}

void tso_export(void* h, const uint32_t* lo, const int32_t* size, float* dist, float* weight, uint8_t* on)
{
    const Tsdm& t = *(Tsdm*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                const Tsd* c = t.get(Vec3u{lo[0] + x, lo[1] + y, lo[2] + z});
                dist[i] = c ? c->distance : 0.f;
                weight[i] = c ? c->weight : 0.f;
                on[i] = c != nullptr;
            }
}

size_t tso_mesh(void* h, float* out, size_t cap)
{
    std::vector<float> v;
    ((Tsdm*)h)->to_mesh(v);
    const size_t n = v.size() / 3;
    if (out && cap >= n) std::copy(v.begin(), v.end(), out);
    return n;
}

// sdm::export_to_ply (export.cpp:112-143)
int tso_write_ply(void* h, const char* path)
{
    std::vector<float> v;
    ((Tsdm*)h)->to_mesh(v);
    const size_t n = v.size() / 3;
    FILE* f = std::fopen(path, "w");
    if (!f) return 0;
    std::fprintf(f, "ply\nformat ascii 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\nelement face %zu\n"
                    "property list uchar int vertex_index\nend_header\n", n, n / 3);
    for (size_t i = 0; i < n; ++i) std::fprintf(f, "%f %f %f\n", v[3 * i], v[3 * i + 1], v[3 * i + 2]);
    for (size_t i = 0; i < n; i += 3) std::fprintf(f, "3 %d %d %d\n", (int)(i + 2), (int)(i + 1), (int)i);
    std::fclose(f);
    return 1;
}

void tso_mc_table(int8_t* tri, uint8_t* ntri)
{
    const McTable t = mc_build_table();
    std::copy(&t.tri[0][0], &t.tri[0][0] + 256 * kMcRow, tri);
    std::copy(t.ntri, t.ntri + 256, ntri);
}
int tso_mc_row() { return kMcRow; }

}  // extern "C"
