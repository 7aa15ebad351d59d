// occ_dist3_emu.cpp -- host build of the coupled insertion (OccMap3Dev::insert_point_clouds_dm3, om3d.cu) on plain host stores: the
// same admission (window margin R + 1, Dm3Guard::admit_entries), the same records cut into the same chunks (a record cap set at
// creation), a stable sort by cell, the per-cell fold through od3_record (occ_dist3_core.h), the distance map's patches allocated in
// ascending entry order, and the op list applied and updated cloud by cloud through Brushfire3::run_segments (ddm3_core.h) with the
// device map's resume loop.  The hooks LAMA_DM3_HEAP_CAP and LAMA_DM3_POP_BUDGET are read at creation, as the device map reads them.
// TEST INFRASTRUCTURE ONLY: compiled by tests/test_occ_dist3d.py into the check binary (occ_dist3_check.cpp), -ffp-contract=off.
#include "../../iris_lama_b200/csrc/occ_dist3_core.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

using namespace lama_b200;

namespace {

// the Map policy of Brushfire3 on a host pool; patches are allocated by the brushfire (first touch) or by alloc()
struct HostDist {
    PatchWindow win{};
    std::vector<int32_t> dir;
    std::vector<std::unique_ptr<uint64_t[]>> slots;
    uint32_t pool = 0, used = 0, err = 0;
    uint64_t scratch = 0;

    void alloc(int di)
    {
        dir[(size_t)di] = (int32_t)used++;
        slots.emplace_back(new uint64_t[kDm3Cells]());
    }
    uint64_t* cell(uint32_t x, uint32_t y, uint32_t z)
    {
        const int di = window_dir_index(win, x, y, z);
        if (di < 0) { err |= kErrWindow; return &scratch; }
        if (dir[(size_t)di] < 0) {
            if (used >= pool) { err |= kErrPoolEmpty; return &scratch; }
            alloc(di);
        }
        uint64_t* p = slots[(size_t)dir[(size_t)di]].get() + dm3_cell_index(x, y, z);
        *p |= kDm3KnownBit;
        return p;
    }
};

uint64_t env_u64(const char* name, uint64_t dflt)
{
    const char* s = std::getenv(name);
    if (!s) return dflt;
    const unsigned long long v = std::strtoull(s, nullptr, 10);
    return v > 0 ? (uint64_t)v : dflt;
}

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

struct Emu {
    int kind = 0;
    double scale = 0;
    ProbParams pp{};
    PatchWindow win{};
    uint64_t record_cap = 0;
    // occupancy map: slot per entry, words and known bits per slot
    std::vector<int32_t> odir;
    std::vector<std::vector<uint32_t>> ocells;
    std::vector<std::vector<uint8_t>> oknown;
    // distance map
    HostDist dm;
    Dm3Guard guard;
    uint32_t max_sqdist = 0;
    std::vector<uint64_t> rq, lq;
    Dm3State st{};
    uint64_t budget = 0, runs = 0, grows = 0;
    std::vector<uint32_t> pending;
    std::string err;

    // DistMap3Dev::drive: launches until done, doubling a heap whenever a run stops for room
    int drive(const uint32_t* ops, uint32_t n_ops, bool do_update, const uint32_t* seg_end, uint32_t n_seg, uint32_t* processed)
    {
        for (;;) {
            Brushfire3<HostDist> b(dm, Heap{rq.data(), st.raise_size, (uint32_t)rq.size()}, Heap{lq.data(), st.lower_size, (uint32_t)lq.size()}, max_sqdist);
            dm.used = st.used;
            if (seg_end) b.run_segments(st, ops, seg_end, n_seg, budget, processed);
            else b.run(st, ops, n_ops, do_update, budget);
            st.raise_size = b.raise_q.size;
            st.lower_size = b.lower_q.size;
            st.used = dm.used;
            st.err |= b.err | dm.err;
            ++runs;
            if (st.err) { err = "internal: the brushfire left the admitted cells"; return -7; }
            if (st.stop == kDm3Done) break;
            if (st.stop == kDm3NeedRoom) {
                if (st.raise_size + kDm3HeapRoom > rq.size()) { rq.resize(rq.size() * 2); ++grows; }
                if (st.lower_size + kDm3HeapRoom > lq.size()) { lq.resize(lq.size() * 2); ++grows; }
            }
        }
        st.next_op = 0;
        st.seg = 0;
        return 0;
    }

    int insert(const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, bool full, uint64_t* cells,
               uint32_t* processed, uint64_t* counts)
    {
        counts[0] = counts[1] = 0;
        struct Rec { uint32_t key, op; };
        std::vector<Rec> recs;
        std::vector<uint64_t> bound((size_t)n + 1, 0);
        std::vector<uint32_t> marks(odir.size(), 0);
        for (int k = 0; k < n; ++k) {
            const Affine tf = cloud_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr);
            for (int64_t i = offsets[k]; i < offsets[k + 1]; ++i) {
                const BeamCells b = om3_point_cells(tf, pts + 3 * i, scale);
                bool bad = false;
                auto touch = [&](uint32_t x, uint32_t y, uint32_t z, uint32_t op) {
                    const int di = window_dir_index(win, x, y, z);
                    if (di < 0 || !dm3_inside(win, x, y, z, guard.reach + 1)) { bad = true; return; }
                    marks[(size_t)di] = 1;
                    recs.push_back(Rec{((uint32_t)di << kOm3Log2Cells) | window_cell_index(x, y, z, 1), op});
                };
                touch(b.to[0], b.to[1], b.to[2], kOm3SetOccupied);
                if (full) {
                    RayWalk3 w(b);
                    while (w.next() && !bad) touch(w.x, w.y, w.z, kOm3SetFree);
                }
                if (bad) { err = "window"; return -4; }
            }
            bound[(size_t)k + 1] = recs.size();
        }
        for (int k = 0; k < n; ++k)
            if (bound[(size_t)k + 1] - bound[(size_t)k] >= (uint64_t(1) << 30)) { err = "cloud too long"; return -1; }
        std::vector<uint8_t> next;
        if (guard.admit_entries(marks, dm.dir, (int64_t)dm.pool - st.used, next, err) != 0) return -5;
        for (size_t di = 0; di < marks.size(); ++di)
            if (marks[di] && odir[di] < 0) {
                odir[di] = (int32_t)ocells.size();
                ocells.emplace_back((size_t)kOm3Cells, 0u);
                oknown.emplace_back((size_t)kOm3Cells, (uint8_t)0);
            }
        guard.reachable.swap(next);
        if (!pending.empty()) {   // the queued ops, without update()
            const int rc = drive(pending.data(), (uint32_t)(pending.size() / kDm3OpWords), false, nullptr, 0, nullptr);
            if (rc != 0) return rc;
            pending.clear();
        }
        for (int c0 = 0; c0 < n;) {   // PatchStore::for_each_chunk
            int c1 = c0 + 1;
            while (c1 < n && bound[(size_t)c1 + 1] - bound[(size_t)c0] <= record_cap) ++c1;
            const uint64_t base = bound[(size_t)c0], nrec = bound[(size_t)c1] - base;
            std::vector<uint8_t> flags((size_t)nrec, 0);
            std::vector<uint32_t> order((size_t)nrec);
            std::iota(order.begin(), order.end(), 0u);
            std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return recs[base + a].key < recs[base + b].key; });
            for (uint64_t i = 0; i < nrec; ++i) {   // the emit pass's known bits
                const uint32_t key = recs[base + i].key;
                oknown[(size_t)odir[key >> kOm3Log2Cells]][key & (kOm3Cells - 1)] = 1;
            }
            for (uint64_t i = 0; i < nrec;) {       // k_od3_fold
                const uint32_t key = recs[base + order[i]].key, di = key >> kOm3Log2Cells, ci = key & (kOm3Cells - 1);
                uint32_t& word = ocells[(size_t)odir[di]][ci];
                const int32_t ds = dm.dir[di];
                bool obstacle = ds >= 0 && dm3_obstacle(dm.slots[(size_t)ds][ci]);
                for (; i < nrec && recs[base + order[i]].key == key; ++i) flags[order[i]] = (uint8_t)od3_record(kind, pp, word, recs[base + order[i]].op, obstacle);
            }
            std::vector<uint32_t> emarks(odir.size(), 0);   // k_od3_mark, then the allocation in ascending entry order
            for (uint64_t i = 0; i < nrec; ++i)
                if (flags[i] & kOd3Event) emarks[recs[base + i].key >> kOm3Log2Cells] = 1;
            for (size_t di = 0; di < emarks.size(); ++di)
                if (emarks[di] && dm.dir[di] < 0) {
                    if (st.used >= dm.pool) { err = "internal: pool"; return -7; }
                    dm.used = st.used;
                    dm.alloc((int)di);
                    st.used = dm.used;
                }
            std::vector<uint32_t> ops, seg_end((size_t)(c1 - c0), 0);
            for (uint64_t i = 0; i < nrec; ++i) {   // k_od3_known and k_od3_ops
                const uint32_t f = flags[i], key = recs[base + i].key;
                if (!(f & kOd3Event)) continue;
                ++counts[0];
                dm.slots[(size_t)dm.dir[key >> kOm3Log2Cells]][key & (kOm3Cells - 1)] |= kDm3KnownBit;
                if (!(f & kOd3Push)) continue;
                uint32_t x, y, z;
                dm3_key_cell(win, key, x, y, z);
                ops.insert(ops.end(), {x, y, z, (f & kOd3Remove) ? 1u : 0u});
            }
            for (int c = c0; c < c1; ++c) {         // k_od3_segments
                uint32_t e = 0;
                for (uint64_t i = 0; i < bound[(size_t)c + 1] - base; ++i) e += (flags[i] & kOd3Push) ? 1u : 0u;
                seg_end[(size_t)(c - c0)] = e;
            }
            counts[1] += ops.size() / kDm3OpWords;
            st.processed = 0;
            st.seg = 0;
            const int rc = drive(ops.data(), (uint32_t)(ops.size() / kDm3OpWords), true, seg_end.data(), (uint32_t)seg_end.size(), processed + c0);
            if (rc != 0) return rc;
            st.processed = 0;
            c0 = c1;
        }
        *cells = bound[(size_t)n];
        return 0;
    }
};

}  // namespace

extern "C" {

// kind 0 frequency / 1 log-odds; window (patches per axis) centred on the origin; dm_pool 0 = one slot per entry; record_cap the
// records of one chunk
void* od3e_create(int kind, double resolution, double l2_max, const int32_t* window, int dm_pool, uint64_t record_cap)
{
    Emu* e = new Emu();
    e->kind = kind;
    e->scale = 1.0 / resolution;
    e->record_cap = record_cap;
    auto logods = [](float prob) -> float { return (float)std::log(prob / (1.0 - prob)); };   // as the device map builds ProbParams
    e->pp.miss = logods(0.4f);
    e->pp.hit = logods(0.7f);
    e->pp.clamp_min = logods(0.12f);
    e->pp.clamp_max = logods(0.97f);
    e->pp.thresh = 0.0 * logods(0.5f);
    PatchWindow& w = e->win;
    w.is3d = 1;
    for (int k = 0; k < 3; ++k) {
        w.dim[k] = window[k];
        w.base[k] = (int32_t)(w2m(0.0, e->scale) >> kPatchLog2) - window[k] / 2;
    }
    const size_t ndir = (size_t)w.dim[0] * w.dim[1] * w.dim[2];
    e->odir.assign(ndir, -1);
    e->dm.win = w;
    e->dm.dir.assign(ndir, -1);
    e->dm.pool = dm_pool > 0 ? (uint32_t)dm_pool : (uint32_t)ndir;
    const uint32_t r = (uint32_t)std::ceil(l2_max * e->scale);
    e->max_sqdist = r * r;
    e->guard.init(w, (int)r);
    const uint64_t cap = env_u64("LAMA_DM3_HEAP_CAP", uint64_t(1) << 16);
    e->rq.assign(cap, 0);
    e->lq.assign(cap, 0);
    e->budget = env_u64("LAMA_DM3_POP_BUDGET", uint64_t(1) << 20);
    return e;
}
void od3e_destroy(void* h) { delete (Emu*)h; }
const char* od3e_error(void* h) { return ((Emu*)h)->err.c_str(); }

// addObstacle (remove = 0) / removeObstacle of n cells, admitted and queued as DistMap3Dev::add_remove does; 0, -4 or -5
int od3e_queue(void* h, const uint32_t* xyz, int n, int remove)
{
    Emu& e = *(Emu*)h;
    const int rc = e.guard.admit(xyz, n, 3, e.dm.dir, (int64_t)e.dm.pool - e.st.used, e.err);
    if (rc != 0) return rc;
    for (int i = 0; i < n; ++i) e.pending.insert(e.pending.end(), {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], remove ? 1u : 0u});
    return 0;
}

// the coupled insertion; 0, -1, -4, -5 or -7 (internal)
int od3e_update_maps(void* h, const double* pts, const int64_t* offsets, int n, const double* origins, const double* quats, int full, uint64_t* cells,
                     uint32_t* processed, uint64_t* counts)
{
    return ((Emu*)h)->insert(pts, offsets, n, origins, quats, full != 0, cells, processed, counts);
}

// the box lo + [0, size), x fastest: occupancy words and known bits
void od3e_om_export(void* h, const uint32_t* lo, const int32_t* size, uint32_t* words, uint8_t* known)
{
    const Emu& e = *(Emu*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                const uint32_t cx = lo[0] + x, cy = lo[1] + y, cz = lo[2] + z;
                const int di = window_dir_index(e.win, cx, cy, cz);
                const int32_t s = di < 0 ? -1 : e.odir[(size_t)di];
                const uint32_t ci = window_cell_index(cx, cy, cz, 1);
                known[i] = s < 0 ? 0 : e.oknown[(size_t)s][ci];
                words[i] = known[i] ? e.ocells[(size_t)s][ci] : 0u;
            }
}
// the box lo + [0, size), x fastest: distance words (ddm3_core.h) and known bits
void od3e_dm_export(void* h, const uint32_t* lo, const int32_t* size, uint64_t* words, uint8_t* known)
{
    const Emu& e = *(Emu*)h;
    size_t i = 0;
    for (int z = 0; z < size[2]; ++z)
        for (int y = 0; y < size[1]; ++y)
            for (int x = 0; x < size[0]; ++x, ++i) {
                const uint32_t cx = lo[0] + x, cy = lo[1] + y, cz = lo[2] + z;
                const int di = window_dir_index(e.win, cx, cy, cz);
                const int32_t s = di < 0 ? -1 : e.dm.dir[(size_t)di];
                words[i] = s < 0 ? 0 : e.dm.slots[(size_t)s][dm3_cell_index(cx, cy, cz)];
                known[i] = dm3_known(words[i]);
            }
}
// the patch ids (Map::m2p with is_3d) of the allocated entries of the occupancy (which = 0) or distance map, ascending entry
int od3e_patch_ids(void* h, int which, uint64_t* ids)
{
    const Emu& e = *(Emu*)h;
    const std::vector<int32_t>& dir = which ? e.dm.dir : e.odir;
    int n = 0;
    for (size_t i = 0; i < dir.size(); ++i) {
        if (dir[i] < 0) continue;
        uint32_t a[3];
        window_anchor(e.win, (int)i, a);
        if (ids) ids[n] = ((uint64_t)(a[0] >> kPatchLog2) * 2642244ull + (a[1] >> kPatchLog2)) * 2642244ull + (a[2] >> kPatchLog2);
        ++n;
    }
    return n;
}
// {brushfire runs, heap growths}
void od3e_stats(void* h, uint64_t* out)
{
    out[0] = ((Emu*)h)->runs;
    out[1] = ((Emu*)h)->grows;
}

}  // extern "C"
