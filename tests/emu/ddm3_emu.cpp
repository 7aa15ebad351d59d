// ddm3_emu.cpp -- host build of the 3-D distance map core (iris_lama_b200/csrc/ddm3_core.h): the admission (Dm3Guard), the resumable
// brushfire (Brushfire3::run) and the heap growth between runs, as DistMap3Dev (ddm3d.cu) drives them, on a host pool of 32^3-cell
// slots taken in first-touch order, for comparison with the oracle (ddm3_oracle.cpp).  The test hooks LAMA_DM3_HEAP_CAP (initial
// heap capacity) and LAMA_DM3_POP_BUDGET (pops per run) are read at creation, as the device map reads them.
// TEST INFRASTRUCTURE ONLY: compiled by tests/ddm3_oracle.py, -ffp-contract=off (and by the sanitizer build of ddm3_check.cpp).
#include "../../iris_lama_b200/csrc/ddm3_core.h"

#include <cmath>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

using namespace lama_b200;

namespace {

struct HostMap3 {
    PatchWindow win{};
    std::vector<int32_t> dir;
    std::vector<std::unique_ptr<uint64_t[]>> slots;
    uint32_t pool = 0, used = 0, err = 0;
    uint64_t scratch = 0;

    uint64_t* cell(uint32_t x, uint32_t y, uint32_t z)
    {
        const int di = window_dir_index(win, x, y, z);
        if (di < 0) { err |= kErrWindow; return &scratch; }
        int32_t slot = dir[(size_t)di];
        if (slot < 0) {
            if (used >= pool) { err |= kErrPoolEmpty; return &scratch; }
            slot = (int32_t)used++;
            dir[(size_t)di] = slot;
            slots.emplace_back(new uint64_t[kDm3Cells]());
        }
        uint64_t* p = slots[(size_t)slot].get() + dm3_cell_index(x, y, z);
        *p |= kDm3KnownBit;
        return p;
    }
    const uint64_t* peek(uint32_t x, uint32_t y, uint32_t z) const   // the const get: null when absent or unknown
    {
        const int di = window_dir_index(win, x, y, z);
        if (di < 0 || dir[(size_t)di] < 0) return nullptr;
        const uint64_t* p = slots[(size_t)dir[(size_t)di]].get() + dm3_cell_index(x, y, z);
        return dm3_known(*p) ? p : nullptr;
    }
};

uint64_t env_u64(const char* name, uint64_t dflt)
{
    const char* s = std::getenv(name);
    if (!s) return dflt;
    const unsigned long long v = std::strtoull(s, nullptr, 10);
    return v > 0 ? (uint64_t)v : dflt;
}

struct Emu {
    double resolution = 0, scale = 0;
    uint32_t max_sqdist = 0;
    HostMap3 map;
    Dm3Guard guard;
    std::vector<uint64_t> rq, lq;   // heap storage; the capacity is the size
    Dm3State st{};
    std::vector<uint32_t> pending;
    uint64_t budget = 0;
    uint64_t runs = 0, grows = 0;
    std::string err;

    int run(bool do_update, uint32_t* processed)
    {
        st.next_op = 0;
        if (do_update) st.processed = 0;
        const uint32_t n_ops = (uint32_t)(pending.size() / kDm3OpWords);
        for (;;) {
            Brushfire3<HostMap3> b(map, Heap{rq.data(), st.raise_size, (uint32_t)rq.size()}, Heap{lq.data(), st.lower_size, (uint32_t)lq.size()}, max_sqdist);
            map.used = st.used;
            b.run(st, pending.data(), n_ops, do_update, budget);
            st.raise_size = b.raise_q.size;
            st.lower_size = b.lower_q.size;
            st.used = map.used;
            st.err |= b.err | map.err;
            ++runs;
            if (st.err) { err = "internal: the brushfire left the admitted cells"; return -7; }
            if (st.stop == kDm3Done) break;
            if (st.stop == kDm3NeedRoom) {
                if (st.raise_size + kDm3HeapRoom > rq.size()) { rq.resize(rq.size() * 2); ++grows; }
                if (st.lower_size + kDm3HeapRoom > lq.size()) { lq.resize(lq.size() * 2); ++grows; }
            }
        }
        pending.clear();
        if (processed) *processed = st.processed;
        return 0;
    }
    int flush() { return pending.empty() ? 0 : run(false, nullptr); }
    double cell_distance(uint32_t x, uint32_t y, uint32_t z) const   // dynamic_distance_map.cpp:140-147
    {
        const uint64_t* c = map.peek(x, y, z);
        return sqrt((double)(c && dm3_valid(*c) ? dm3_sqdist(*c) : max_sqdist)) * resolution;
    }
};

}  // namespace

extern "C" {

// window (patches per axis) centred on center (cells); pool_slots 0 = one per entry
void* d3e_create(double resolution, double l2_max, const double* center, const int32_t* window, int pool_slots)
{
    Emu* e = new Emu();
    e->resolution = resolution;
    e->scale = 1.0 / resolution;
    const uint32_t r = (uint32_t)std::ceil(l2_max * e->scale);
    e->max_sqdist = r * r;
    PatchWindow& w = e->map.win;
    w.is3d = 1;
    for (int k = 0; k < 3; ++k) {
        w.dim[k] = window[k];
        w.base[k] = (int32_t)(w2m(center ? center[k] : 0.0, e->scale) >> kPatchLog2) - window[k] / 2;
    }
    const size_t ndir = (size_t)w.dim[0] * w.dim[1] * w.dim[2];
    e->map.dir.assign(ndir, -1);
    e->map.pool = pool_slots > 0 ? (uint32_t)pool_slots : (uint32_t)ndir;
    e->guard.init(w, (int)r);
    const uint64_t cap = env_u64("LAMA_DM3_HEAP_CAP", uint64_t(1) << 16);
    e->rq.assign(cap, 0);
    e->lq.assign(cap, 0);
    e->budget = env_u64("LAMA_DM3_POP_BUDGET", uint64_t(1) << 20);
    return e;
}
void d3e_destroy(void* h) { delete (Emu*)h; }
const char* d3e_error(void* h) { return ((Emu*)h)->err.c_str(); }

// the host admission of n ops (x, y, z, kind), then queued; 0, -4 (window) or -5 (pool), the map unchanged on a refusal
int d3e_apply(void* h, const uint32_t* ops, int n)
{
    Emu& e = *(Emu*)h;
    const int rc = e.guard.admit(ops, n, kDm3OpWords, e.map.dir, (int64_t)e.map.pool - e.st.used, e.err);
    if (rc != 0) return rc;
    e.pending.insert(e.pending.end(), ops, ops + (size_t)kDm3OpWords * n);
    return 0;
}
int d3e_update(void* h, uint32_t* processed) { return ((Emu*)h)->run(true, processed); }

void d3e_distance(void* h, const double* pts, int n, double* dist, double* grad)
{
    Emu& e = *(Emu*)h;
    e.flush();
    for (int i = 0; i < n; ++i) {
        double g[3];
        dist[i] = trilinear_distance(pts + 3 * i, e.scale, [&](uint32_t x, uint32_t y, uint32_t z) { return e.cell_distance(x, y, z); }, g);
        if (grad) for (int k = 0; k < 3; ++k) grad[3 * i + k] = g[k];
    }
}
void d3e_cell_distance(void* h, const uint32_t* xyz, int n, double* dist)
{
    Emu& e = *(Emu*)h;
    e.flush();
    for (int i = 0; i < n; ++i) dist[i] = e.cell_distance(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}
int d3e_bounds(void* h, uint32_t* mn, uint32_t* mx)
{
    Emu& e = *(Emu*)h;
    e.flush();
    int n = 0;
    for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0; }
    for (size_t i = 0; i < e.map.dir.size(); ++i) {
        if (e.map.dir[i] < 0) continue;
        uint32_t a[3];
        window_anchor(e.map.win, (int)i, a);
        for (int k = 0; k < 3; ++k) { mn[k] = a[k] < mn[k] ? a[k] : mn[k]; mx[k] = a[k] > mx[k] ? a[k] : mx[k]; }
        ++n;
    }
    for (int k = 0; k < 3; ++k) mx[k] += kPatchLen;
    return n;
}
void d3e_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known)
{
    Emu& e = *(Emu*)h;
    e.flush();
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                const uint32_t cx = lo[0] + x, cy = lo[1] + y, cz = lo[2] + z;
                const int di = window_dir_index(e.map.win, cx, cy, cz);
                const int32_t slot = di < 0 ? -1 : e.map.dir[(size_t)di];
                const uint64_t w = slot < 0 ? 0 : e.map.slots[(size_t)slot][dm3_cell_index(cx, cy, cz)];
                words[i] = w;
                known[i] = dm3_known(w);
            }
}
// the patch ids (Map::m2p with is_3d, map.h:153-161) of the allocated entries, ascending entry
int d3e_patch_ids(void* h, uint64_t* ids)
{
    Emu& e = *(Emu*)h;
    e.flush();
    int n = 0;
    for (size_t i = 0; i < e.map.dir.size(); ++i) {
        if (e.map.dir[i] < 0) continue;
        uint32_t a[3];
        window_anchor(e.map.win, (int)i, a);
        ids[n++] = ((uint64_t)(a[0] >> kPatchLog2) * 2642244ull + (a[1] >> kPatchLog2)) * 2642244ull + (a[2] >> kPatchLog2);
    }
    return n;
}
// {runs, heap growths, raise capacity, lower capacity}
void d3e_stats(void* h, uint64_t* out)
{
    const Emu& e = *(Emu*)h;
    out[0] = e.runs;
    out[1] = e.grows;
    out[2] = e.rq.size();
    out[3] = e.lq.size();
}

}  // extern "C"
