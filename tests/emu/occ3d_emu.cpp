// occ3d_emu.cpp -- host build of the 3-D occupancy core (iris_lama_b200/csrc/om3d_core.h): insertion and the ordered setters run
// sequentially through the same om3_point_cells / RayWalk3 / om3_op / om3_flags calls as the device kernels (om3d.cu), on a plain
// host store, for comparison with the oracle (occ3d_oracle.cpp).
// TEST INFRASTRUCTURE ONLY: compiled by tests/occ3d_oracle.py, -ffp-contract=off.
#include "../../iris_lama_b200/csrc/om3d_core.h"

#include <cmath>
#include <map>
#include <tuple>

using namespace lama_b200;

namespace {

using Key = std::tuple<uint32_t, uint32_t, uint32_t>;

struct Emu {
    int kind;
    double scale;
    ProbParams pp;
    std::map<Key, uint32_t> cells;   // known cells and their words

    bool op(uint32_t x, uint32_t y, uint32_t z, uint32_t o) { return om3_op(kind, cells[Key(x, y, z)], o, pp); }   // Map::get sets the bit
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

void* o3e_create(double resolution, int kind)
{
    Emu* e = new Emu();
    e->kind = kind;
    e->scale = 1.0 / resolution;
    auto logods = [](float prob) -> float { return (float)std::log(prob / (1.0 - prob)); };   // as the device map builds ProbParams
    e->pp.miss = logods(0.4f);
    e->pp.hit = logods(0.7f);
    e->pp.clamp_min = logods(0.12f);
    e->pp.clamp_max = logods(0.97f);
    e->pp.thresh = 0.0 * logods(0.5f);
    return e;
}
void o3e_destroy(void* h) { delete (Emu*)h; }

uint64_t o3e_insert(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, int full)
{
    Emu& e = *(Emu*)h;
    uint64_t cells = 0;
    for (int k = 0; k < n; ++k) {
        const Affine a = cloud_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
        for (int64_t i = offsets[k]; i < offsets[k + 1]; ++i) {
            const BeamCells b = om3_point_cells(a, pts + 3 * i, e.scale);
            cells += om3_point_records(b, full != 0);
            e.op(b.to[0], b.to[1], b.to[2], kOm3SetOccupied);
            if (!full) continue;
            RayWalk3 w(b);
            while (w.next()) e.op(w.x, w.y, w.z, kOm3SetFree);
        }
    }
    return cells;
}

void o3e_apply(void* h, const uint32_t* xyz, const uint8_t* ops, int n, uint8_t* changed)
{
    Emu& e = *(Emu*)h;
    for (int i = 0; i < n; ++i) {
        const bool r = e.op(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], ops[i]);
        if (changed) changed[i] = r;
    }
}

void o3e_query(void* h, const uint32_t* xyz, int n, double* prob, uint8_t* flags)
{
    const Emu& e = *(Emu*)h;
    auto prob_of = [](float l) -> float { return 1.0 - 1.0 / (1.0 + std::exp(l)); };
    for (int i = 0; i < n; ++i) {
        auto it = e.cells.find(Key(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
        const bool known = it != e.cells.end();
        const uint32_t w = known ? it->second : 0u;
        flags[i] = (uint8_t)om3_flags(e.kind, known, w, e.pp);
        if (e.kind == kOm3Frequency) prob[i] = occ_visited(w) == 0 ? 0.25 : (double)occ_occupied(w) / (double)occ_visited(w);
        else prob[i] = prob_of(known ? om3_bits_float(w) : (float)e.pp.thresh);
    }
}

void o3e_prune(void* h)
{
    for (auto& kv : ((Emu*)h)->cells) kv.second = om3_prune(kv.second);
}

void o3e_export(void* h, const uint32_t* lo, const int32_t* size, uint32_t* words, uint8_t* known)
{
    const Emu& e = *(Emu*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                auto it = e.cells.find(Key(lo[0] + x, lo[1] + y, lo[2] + z));
                known[i] = it != e.cells.end();
                words[i] = known[i] ? it->second : 0u;
            }
}

}  // extern "C"
