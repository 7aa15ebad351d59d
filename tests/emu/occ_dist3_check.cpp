// occ_dist3_check.cpp -- a standalone comparison of the host build of the coupled insertion (occ_dist3_emu.cpp) with the oracle
// composition (occ_dist3_oracle.cpp over occ3d_oracle.cpp and ddm3_oracle.cpp) on one scenario file, built with and without
// -fsanitize=address,undefined by tests/test_occ_dist3d.py.  Exit status 0 when every comparison holds.
//   usage: occ_dist3_check <scenario>
// The scenario is little-endian float64 values: kind, resolution, l2_max, record_cap, wx, wy, wz, dm_pool, full, n_batches, then per
// batch: n_queued, n_queued cells (x y z, queued addObstacles before the call), n_clouds, and per cloud: origin (3), quaternion xyzw
// (4), n_points, the points (3 each).  After every batch both sides must agree on the cell updates, processed per cloud, the event
// and push counts, both patch sets and bounds, and every cell of every patch of both maps.
// TEST INFRASTRUCTURE ONLY.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <vector>

extern "C" {
void* o3o_create(double resolution, int kind);
void o3o_destroy(void* h);
int o3o_bounds(void* h, uint32_t* mn, uint32_t* mx);
void o3o_export(void* h, const uint32_t* lo, const int32_t* size, uint32_t* words, uint8_t* known);
void* d3o_create(double resolution, double l2_max);
void d3o_destroy(void* h);
void d3o_apply(void* h, const uint32_t* ops, int n);
int d3o_bounds(void* h, uint32_t* mn, uint32_t* mx);
int d3o_patch_ids(void* h, uint64_t* ids);
void d3o_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known);
uint64_t od3o_update_maps(void* om, void* dm, double resolution, const double* pts, const int64_t* offsets, int n, const double* origins,
                          const double* quats, int full, uint32_t* processed, uint64_t* counts);
void* od3e_create(int kind, double resolution, double l2_max, const int32_t* window, int dm_pool, uint64_t record_cap);
void od3e_destroy(void* h);
const char* od3e_error(void* h);
int od3e_queue(void* h, const uint32_t* xyz, int n, int remove);
int od3e_update_maps(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, int full, uint64_t* cells,
                     uint32_t* processed, uint64_t* counts);
void od3e_om_export(void* h, const uint32_t* lo, const int32_t* size, uint32_t* words, uint8_t* known);
void od3e_dm_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known);
int od3e_patch_ids(void* h, int which, uint64_t* ids);
}

namespace {

const uint64_t kUc = 2642244ull, kUc2 = kUc * kUc;

void anchor(uint64_t id, uint32_t lo[3])
{
    lo[0] = (uint32_t)((id / kUc2) << 5);
    lo[1] = (uint32_t)(((id % kUc2) / kUc) << 5);
    lo[2] = (uint32_t)((id % kUc) << 5);
}

// both maps of both sides after batch b; false (with a message) at the first difference
bool same(void* om, void* dm, void* e, int b)
{
    const int32_t size[3] = {32, 32, 32};
    uint32_t mno[3], mxo[3];
    // occupancy: the emulation's patches; the oracle has as many, and every emulated patch has a known cell, so the sets are equal
    // when every emulated patch's cells are
    std::vector<uint64_t> ie((size_t)od3e_patch_ids(e, 0, nullptr));
    od3e_patch_ids(e, 0, ie.data());
    if (o3o_bounds(om, mno, mxo) != (int)ie.size()) { std::fprintf(stderr, "batch %d: occupancy patch counts differ\n", b); return false; }
    std::vector<uint32_t> wo(32768), we(32768);
    std::vector<uint8_t> ko(32768), ke(32768);
    for (uint64_t id : ie) {
        uint32_t lo[3];
        anchor(id, lo);
        o3o_export(om, lo, size, wo.data(), ko.data());
        od3e_om_export(e, lo, size, we.data(), ke.data());
        if (wo != we || ko != ke) { std::fprintf(stderr, "batch %d: occupancy cells of patch %llu differ\n", b, (unsigned long long)id); return false; }
    }
    // distance map
    const int no = d3o_bounds(dm, mno, mxo);
    std::vector<uint64_t> io((size_t)no), je((size_t)od3e_patch_ids(e, 1, nullptr));
    d3o_patch_ids(dm, io.data());
    od3e_patch_ids(e, 1, je.data());
    if (std::set<uint64_t>(io.begin(), io.end()) != std::set<uint64_t>(je.begin(), je.end())) {
        std::fprintf(stderr, "batch %d: distance patch sets differ (%zu, %zu)\n", b, io.size(), je.size());
        return false;
    }
    std::vector<uint64_t> xo(32768), xe(32768);
    for (uint64_t id : io) {
        uint32_t lo[3];
        anchor(id, lo);
        d3o_export(dm, lo, size, xo.data(), ko.data());
        od3e_dm_export(e, lo, size, xe.data(), ke.data());
        if (xo != xe || ko != ke) { std::fprintf(stderr, "batch %d: distance cells of patch %llu differ\n", b, (unsigned long long)id); return false; }
    }
    return true;
}

}  // namespace

int main(int argc, char** argv)
{
    if (argc != 2) { std::fprintf(stderr, "usage: occ_dist3_check <scenario>\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<double> s;
    double v;
    while (std::fread(&v, 8, 1, f) == 1) s.push_back(v);
    std::fclose(f);
    if (s.size() < 10) return 2;
    size_t at = 0;
    auto next = [&]() { return at < s.size() ? s[at++] : (std::fprintf(stderr, "short scenario\n"), std::exit(2), 0.0); };
    const int kind = (int)next();
    const double res = next(), l2 = next();
    const uint64_t cap = (uint64_t)next();
    int32_t win[3];
    for (int k = 0; k < 3; ++k) win[k] = (int32_t)next();
    const int pool = (int)next(), full = (int)next(), n_batches = (int)next();
    void* om = o3o_create(res, kind);
    void* dm = d3o_create(res, l2);
    void* e = od3e_create(kind, res, l2, win, pool, cap);
    int bad = 0, b = 0;
    for (; b < n_batches && !bad; ++b) {
        const int nq = (int)next();
        std::vector<uint32_t> q((size_t)nq * 3), qo;
        for (auto& c : q) c = (uint32_t)next();
        for (int i = 0; i < nq; ++i) qo.insert(qo.end(), {q[3 * i], q[3 * i + 1], q[3 * i + 2], 0u});
        if (nq && od3e_queue(e, q.data(), nq, 0) != 0) { std::fprintf(stderr, "batch %d: queue refused: %s\n", b, od3e_error(e)); bad = 1; break; }
        d3o_apply(dm, qo.data(), nq);
        const int nc = (int)next();
        std::vector<double> origins, quats, pts;
        std::vector<int64_t> offsets(1, 0);
        for (int c = 0; c < nc; ++c) {
            for (int k = 0; k < 3; ++k) origins.push_back(next());
            for (int k = 0; k < 4; ++k) quats.push_back(next());
            const int64_t np = (int64_t)next();
            for (int64_t i = 0; i < 3 * np; ++i) pts.push_back(next());
            offsets.push_back(offsets.back() + np);
        }
        std::vector<uint32_t> po((size_t)nc), pe((size_t)nc);
        uint64_t co[2], ce[2], cells_e = 0;
        const uint64_t cells_o = od3o_update_maps(om, dm, res, pts.data(), offsets.data(), nc, origins.data(), quats.data(), full, po.data(), co);
        const int rc = od3e_update_maps(e, pts.data(), offsets.data(), nc, origins.data(), quats.data(), full, &cells_e, pe.data(), ce);
        if (rc != 0) { std::fprintf(stderr, "batch %d: rc %d: %s\n", b, rc, od3e_error(e)); bad = 1; break; }
        if (cells_o != cells_e || po != pe || co[0] != ce[0] || co[1] != ce[1]) {
            std::fprintf(stderr, "batch %d: cells %llu/%llu events %llu/%llu pushes %llu/%llu or processed differ\n", b, (unsigned long long)cells_o,
                         (unsigned long long)cells_e, (unsigned long long)co[0], (unsigned long long)ce[0], (unsigned long long)co[1], (unsigned long long)ce[1]);
            bad = 1;
            break;
        }
        if (!same(om, dm, e, b)) { bad = 1; break; }
        std::printf("batch %d: %llu cells, %llu events, %llu pushes\n", b, (unsigned long long)cells_o, (unsigned long long)co[0], (unsigned long long)co[1]);
    }
    o3o_destroy(om);
    d3o_destroy(dm);
    od3e_destroy(e);
    if (!bad) std::printf("ok: %d batches\n", b);
    return bad;
}
