// tsdm_emu.cpp -- host build of the device fusion core (iris_lama_b200/csrc/tsdm_core.h): the same tsdm_ray / RayWalk3 /
// tsdm_sample / tsdm_fold calls as k_tsdm_walk and k_fold_runs, run sequentially on a plain host store, for comparison with the
// oracle (tsdm_oracle.cpp).  TEST INFRASTRUCTURE ONLY: compiled by tests/tsdm_oracle.py, -ffp-contract=off.
#include "../../iris_lama_b200/csrc/mc_table.h"
#include "../../iris_lama_b200/csrc/tsdm_core.h"

#include <cstring>
#include <map>
#include <set>
#include <tuple>
#include <vector>

using namespace lama_b200;

namespace {

struct Cell {
    float d = 0, w = 0;
};

struct Emu {
    TsdmParams prm;
    std::map<std::tuple<uint32_t, uint32_t, uint32_t>, Cell> cells;   // "on" cells; z = 0 in 2-D

    std::tuple<uint32_t, uint32_t, uint32_t> key(uint32_t x, uint32_t y, uint32_t z) const { return std::make_tuple(x, y, prm.is3d ? z : 0u); }
    double value(uint32_t x, uint32_t y, uint32_t z) const
    {
        auto it = cells.find(key(x, y, z));
        if (it == cells.end() || it->second.w == 0.0f) return prm.truncate;
        return it->second.d;
    }
};

Affine cloud_tf(const double* origin, const double* quat)
{
    const double x = quat ? quat[0] : 0, y = quat ? quat[1] : 0, z = quat ? quat[2] : 0, w = quat ? quat[3] : 1;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    Affine a;
    a.l[0] = 1 - (tyy + tzz); a.l[1] = txy - twz;       a.l[2] = txz + twy;
    a.l[3] = txy + twz;       a.l[4] = 1 - (txx + tzz); a.l[5] = tyz - twx;
    a.l[6] = txz - twy;       a.l[7] = tyz + twx;       a.l[8] = 1 - (txx + tyy);
    for (int i = 0; i < 3; ++i) a.t[i] = origin ? origin[i] : 0.0;
    return a;
}

}  // namespace

extern "C" {

void* tse_create(double resolution, int is3d)
{
    Emu* e = new Emu();
    e->prm.scale = 1.0 / resolution;
    e->prm.truncate = 0.15f;
    e->prm.delta = (float)(4 * resolution);
    e->prm.epsilon = (float)resolution;
    e->prm.max_weight = 10000.0f;
    e->prm.is3d = is3d;
    return e;
}
void tse_destroy(void* h) { delete (Emu*)h; }

void tse_insert(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, uint64_t* out)
{
    Emu& e = *(Emu*)h;
    for (int k = 0; k < n; ++k) {
        const Affine a = cloud_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
        std::set<std::tuple<uint32_t, uint32_t, uint32_t>> keys;
        for (int64_t i = offsets[k]; i < offsets[k + 1]; ++i) {
            double hit[3];
            apply_tf(a, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], hit);
            if (!keys.insert(std::make_tuple(w2m(hit[0], e.prm.scale), w2m(hit[1], e.prm.scale), w2m(hit[2], e.prm.scale))).second) continue;
            const TsdmRay r = tsdm_ray(a.t, hit, e.prm);
            RayWalk3 w(r.cells);
            while (w.next()) {
                Cell& c = e.cells[e.key(w.x, w.y, w.z)];
                float d, wt;
                if (tsdm_sample(r, w.x, w.y, w.z, e.prm, d, wt)) tsdm_fold(c.d, c.w, d, wt, e.prm.max_weight);
            }
        }
        if (out) out[k] = keys.size();
    }
}

void tse_export(void* h, const uint32_t* lo, const int32_t* size, float* dist, float* weight, uint8_t* on)
{
    const Emu& e = *(Emu*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                auto it = e.cells.find(e.key(lo[0] + x, lo[1] + y, lo[2] + z));
                dist[i] = it == e.cells.end() ? 0.f : it->second.d;
                weight[i] = it == e.cells.end() ? 0.f : it->second.w;
                on[i] = it != e.cells.end();
            }
}

void tse_distance(void* h, const double* pts, int n, double* dist, double* grad)
{
    const Emu& e = *(Emu*)h;
    for (int i = 0; i < n; ++i)
        dist[i] = tsdm_distance(pts + 3 * i, e.prm, [&](uint32_t x, uint32_t y, uint32_t z) { return e.value(x, y, z); }, grad + 3 * i);
}

// the vertices of one cube (mc_cube + mc_edge_vertex with the given table row): -1 when a corner is missing
int tse_cube(void* h, uint32_t x, uint32_t y, uint32_t z, const int8_t* row, float* out)
{
    const Emu& e = *(Emu*)h;
    float pos[8][3], sdf[8];
    auto cell = [&](uint32_t a, uint32_t b, uint32_t c, float& s) {
        auto it = e.cells.find(e.key(a, b, c));
        if (it == e.cells.end() || it->second.w == 0.0f) return false;
        s = it->second.d;
        return true;
    };
    const int config = mc_cube(x, y, z, e.prm.scale, cell, pos, sdf);
    if (config < 0) return -1;
    for (int j = 0; row && row[kMcRow * config + j] != -1; ++j) mc_edge_vertex(row[kMcRow * config + j], pos, sdf, out + 3 * j);
    return config;
}

}  // extern "C"
