// emu.cpp -- TEST-ONLY host emulation of the CUDA kernels' data flow, built from the product's own core headers
// (lama_core.h, ddm_core.h, ray_core.h, match_core.h) so that the `-m "not gpu"` suite exercises the exact logic
// the kernels run: bit-faithful heap, sequential brushfire on packed cells, packed counter updates in an ARBITRARY
// beam order followed by the ordered per-cell replay, and the fused solver control.  Never linked into the product.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <queue>
#include <random>
#include <vector>

#include "../../iris_lama_b200/csrc/ddm_core.h"
#include "../../iris_lama_b200/csrc/match_core.h"
#include "../../iris_lama_b200/csrc/ray_core.h"
#include "../../iris_lama_b200/csrc/ray_pull.h"

using namespace lama_b200;

namespace {

// dense stand-in for directory + patch pool: one word per cell of the window, "known" patches tracked per patch
struct HostMap {
    DirWindow window;
    std::vector<uint32_t> cells;
    std::vector<uint8_t> fbit;   // obstacle-mirror bit plane (StoreView::fbits on the device)
    std::vector<uint8_t> patch_present;
    uint32_t scratch = 0, err = 0;
    int side() const { return window.dim * kPatchLen; }
    void init(const DirWindow& w)
    {
        window = w;
        cells.assign((size_t)side() * side(), 0u);
        fbit.assign((size_t)side() * side(), 0);
        patch_present.assign((size_t)w.dim * w.dim, 0);
    }
    uint32_t* raw(uint32_t x, uint32_t y, bool touch)
    {
        int di = dir_index(window, x, y);
        if (di < 0) { err |= kErrWindow; scratch = 0; return &scratch; }
        if (touch) patch_present[di] = 1;
        uint32_t lx = x - ((uint32_t)window.base_px << kPatchLog2), ly = y - ((uint32_t)window.base_py << kPatchLog2);
        return &cells[(size_t)ly * side() + lx];
    }
};
struct HostDm : HostMap {
    uint32_t* cell(uint32_t x, uint32_t y)  // the mutable Map::get of the distance map
    {
        uint32_t* p = raw(x, y, true);
        if (!(*p & kDmKnown)) *p |= kDmKnown;
        return p;
    }
};

struct Emu {
    double resolution, scale;
    uint32_t max_sqdist;
    HostMap occ;
    HostDm dm;
    std::vector<uint64_t> heap_l, heap_r;
    SE2 pose{1, 0, 0, 0}, odom{1, 0, 0, 0};
    bool has_first = false;
    double trans_thresh = 0.5, rot_thresh = 0.5;
    uint32_t max_iter = 100;
    int strategy = 0;
    uint32_t last_pops = 0, last_cells = 0, last_events = 0, last_log = 0, last_evals = 0, last_iters = 0;
    uint32_t heap_peak[2] = {0, 0};   // largest lower / raise heap size of any brushfire since creation
    bool pull = false;   // map updates through the pull form of the ray cast (ray_pull.h) instead of the per-beam walk
    uint32_t pull_fallbacks = 0;
};

double cell_dist(const Emu& e, uint32_t x, uint32_t y)
{
    HostDm& dm = const_cast<HostDm&>(e.dm);
    int di = dir_index(dm.window, x, y);
    uint32_t w = di < 0 ? 0u : *dm.raw(x, y, false);
    uint32_t sq = (w & kDmValid) ? dm_sqdist(w) : e.max_sqdist;
    return mul_rn(std::sqrt((double)sq), e.resolution);
}

void evaluate(const Emu& e, const ScanParams& sp, const double* pts, const SE2& state, const SolverOptions& so, double meas_sigma, double sums[kNumSums])
{
    for (int k = 0; k < kNumSums; ++k) sums[k] = 0;
    Affine tf = compose_tf(state, sp.moving);
    for (int b = 0; b < sp.n_beams; ++b) {
        double hit[3];
        apply_tf(tf, pts[3 * b], pts[3 * b + 1], pts[3 * b + 2], hit);
        double mx = w2m_nocast(hit[0], sp.scale), my = w2m_nocast(hit[1], sp.scale);
        uint32_t dx = (uint32_t)mx, dy = (uint32_t)my;
        double v[4] = {cell_dist(e, dx, dy), cell_dist(e, dx + 1, dy), cell_dist(e, dx, dy + 1), cell_dist(e, dx + 1, dy + 1)};
        BeamEval be = bilinear(v, add_rn(mx, -(double)dx), add_rn(my, -(double)dy), sp.scale, hit[0], hit[1]);
        accumulate(sums, be, so.robust_kind, so.robust_param, meas_sigma);
    }
}

// k_match: fused solver loop
void solve(Emu& e, const ScanParams& sp, const double* pts, SE2& state, const SolverOptions& so, double sums[kNumSums])
{
    SolverControl ctl;
    ctl.begin(so);
    e.last_evals = 0;
    for (;;) {
        evaluate(e, sp, pts, state, so, 0.05, sums);
        if (ctl.advance(sums, state)) break;
    }
    if (ctl.state_dirty) evaluate(e, sp, pts, state, so, 0.05, sums);
    e.last_evals = ctl.evals_ref;
    e.last_iters = ctl.iter;
}

void run_brushfire(Emu& e, std::vector<uint64_t>& events, uint32_t cells, uint32_t log_size);
bool update_maps_pull(Emu& e, const ScanParams& sp, const double* pts, const SE2& pose);

// k_raycast + k_brushfire; beams are processed in a shuffled order to prove order independence of the design
void update_maps(Emu& e, const ScanParams& sp, const double* pts, const SE2& pose, uint32_t shuffle_seed)
{
    if (e.pull) {
        if (update_maps_pull(e, sp, pts, pose)) return;
        ++e.pull_fallbacks;
    }
    const DirWindow win = e.occ.window;
    Affine tf = compose_tf(pose, sp.moving);
    std::vector<int> order(sp.n_beams);
    for (int i = 0; i < sp.n_beams; ++i) order[i] = i;
    if (shuffle_seed) {
        std::mt19937 g(shuffle_seed);
        std::shuffle(order.begin(), order.end(), g);
    }
    // phase 1: hit-cell set
    std::vector<uint32_t> hitset;
    for (int b = 0; b < sp.n_beams; ++b) {
        BeamCells bc = beam_cells(tf, sp, pts + 3 * b);
        if (bc.mark_hit && dir_index(win, bc.to[0], bc.to[1]) >= 0) hitset.push_back(cell_key(win, bc.to[0], bc.to[1]));
    }
    std::sort(hitset.begin(), hitset.end());
    // phase 3: packed counter updates + candidate log
    std::vector<uint64_t> log;
    uint32_t cells = 0;
    for (int b : order) {
        BeamCells bc = beam_cells(tf, sp, pts + 3 * b);
        if (bc.mark_hit && dir_index(win, bc.to[0], bc.to[1]) >= 0) {
            ++cells;
            *e.occ.raw(bc.to[0], bc.to[1], true) += kOccHitInc;
            log.push_back(log_record(cell_key(win, bc.to[0], bc.to[1]), (uint32_t)b, 0u, true));
        }
        RayWalk w(bc);
        uint32_t pos = 0;
        while (w.next()) {
            ++pos;
            if (dir_index(win, w.x, w.y) < 0) continue;
            ++cells;
            uint32_t* c = e.occ.raw(w.x, w.y, true);
            *c += kOccMissInc;
            uint32_t key = cell_key(win, w.x, w.y);
            const bool obst = e.occ.fbit[c - e.occ.cells.data()] != 0;
            if (obst || std::binary_search(hitset.begin(), hitset.end(), key)) log.push_back(log_record(key, (uint32_t)b, pos, false));
        }
    }
    // phase 4-6: sort, replay per cell, order the events
    std::sort(log.begin(), log.end());
    std::vector<uint64_t> events;
    for (size_t i = 0; i < log.size();) {
        size_t j = i + 1;
        while (j < log.size() && log_key(log[j]) == log_key(log[i])) ++j;
        uint32_t key = log_key(log[i]);
        uint32_t* c = e.occ.raw(key_x(win, key), key_y(win, key), false);
        uint8_t& fb = e.occ.fbit[c - e.occ.cells.data()];
        fb = replay_cell(log.data(), (int)i, (int)j, *c, fb != 0, [&](bool add, uint32_t seq) { events.push_back(push_record((seq << 1) | (add ? 1u : 0u), key)); });
        i = j;
    }
    run_brushfire(e, events, cells, (uint32_t)log.size());
}

void note_heap_peak(Emu& e, const Brushfire<HostDm>& bf)
{
    e.heap_peak[0] = std::max(e.heap_peak[0], bf.lower_q.peak);
    e.heap_peak[1] = std::max(e.heap_peak[1], bf.raise_q.peak);
}

void run_brushfire(Emu& e, std::vector<uint64_t>& events, uint32_t cells, uint32_t log_size)
{
    const DirWindow win = e.occ.window;
    std::sort(events.begin(), events.end());
    // k_brushfire
    e.heap_l.assign(1 << 16, 0);
    e.heap_r.assign(1 << 16, 0);
    Brushfire<HostDm> bf(e.dm, Heap{e.heap_r.data(), 0u, (uint32_t)e.heap_r.size()}, Heap{e.heap_l.data(), 0u, (uint32_t)e.heap_l.size()}, e.max_sqdist);
    for (uint64_t ev : events) {
        uint32_t key = (uint32_t)ev;
        if ((ev >> 32) & 1u) bf.add_obstacle(key_x(win, key), key_y(win, key));
        else bf.remove_obstacle(key_x(win, key), key_y(win, key));
    }
    e.last_pops   = bf.update();
    note_heap_peak(e, bf);
    e.last_cells  = cells;
    e.last_events = (uint32_t)events.size();
    e.last_log    = log_size;
}


// ---- the pull form of the ray cast (ray_pull.h), laid out like k_ray_setup + k_ray_pull --------------------------------------
struct PullScan {
    uint32_t ox = 0, oy = 0;                 // window-relative origin cell
    std::vector<PullEntry> list;             // class lists sorted by (class, slope, beam)
    int prefix[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<uint32_t> hits;              // pull_hit_record, grouped by patch (hit_lo / hit_n per directory entry), unordered inside
    std::vector<int> hit_lo, hit_n;
    std::vector<uint8_t> marked;             // per directory entry
    uint32_t cells = 0;
};

// k_ray_setup: from the window-relative end cells of the beams (all starting in (ox, oy))
void pull_setup(PullScan& ps, uint32_t ox, uint32_t oy, const std::vector<uint32_t>& tx, const std::vector<uint32_t>& ty, const std::vector<uint8_t>& mark_hit, int dim)
{
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= dim) ++log2dim;
    ps.ox = ox; ps.oy = oy;
    ps.marked.assign((size_t)dim * dim, 0);
    ps.hit_lo.assign((size_t)dim * dim, 0);
    ps.hit_n.assign((size_t)dim * dim, 0);
    std::vector<std::pair<uint32_t, uint32_t>> hit_of;   // (directory entry, record)
    std::vector<uint64_t> keys;
    std::vector<uint32_t> nd_of_beam(tx.size(), 0u);
    for (size_t b = 0; b < tx.size(); ++b) {
        const int ex = (int)tx[b] - (int)ox, ey = (int)ty[b] - (int)oy;
        const PullBeam pb = pull_classify(ex, ey);
        if (mark_hit[b]) {
            const uint32_t di = ((ty[b] >> kPatchLog2) << log2dim) | (tx[b] >> kPatchLog2);
            hit_of.push_back({di, pull_hit_record(cell_index(tx[b], ty[b]), (uint32_t)b)});
            ps.marked[di] = 1;
            ps.cells += 1;
        }
        if (pb.n >= 2) {
            ps.cells += pb.n - 1;
            keys.push_back(pull_sort_key(pb.cls, pb.n, pb.d, (uint32_t)b));
            nd_of_beam[b] = pull_pack(pb.n, pb.d);
            pull_mark_beam(ox, oy, ex, ey, [&](int px, int py) { ps.marked[((size_t)py << log2dim) | (size_t)px] = 1; });
        }
    }
    std::sort(keys.begin(), keys.end());
    // counting sort by patch; the order inside a patch is whatever the scatter's atomics produce on the device: scramble it here
    std::mt19937 g(12345u + (uint32_t)tx.size());
    std::shuffle(hit_of.begin(), hit_of.end(), g);
    std::stable_sort(hit_of.begin(), hit_of.end(), [](const std::pair<uint32_t, uint32_t>& l, const std::pair<uint32_t, uint32_t>& r) { return l.first < r.first; });
    for (size_t i = 0; i < hit_of.size(); ++i) {
        if (ps.hit_n[hit_of[i].first]++ == 0) ps.hit_lo[hit_of[i].first] = (int)i;
        ps.hits.push_back(hit_of[i].second);
    }
    int count[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint64_t k : keys) {
        const uint32_t nd = nd_of_beam[pull_key_beam(k)];
        ps.list.push_back(PullEntry{nd, pull_key_beam(k), pull_magic(nd & 0xFFFFu)});
        ++count[pull_key_class(k)];
    }
    for (int c = 0; c < 8; ++c) ps.prefix[c + 1] = ps.prefix[c] + count[c];
}

// the count tile of one patch the way a warp of k_ray_pull fills it: per class every lane runs over the same beam range and drops
// each beam into the counter of the cell where it crosses the lane's column (x-major classes) / row (y-major classes)
void pull_patch_counts(const PullScan& ps, int px, int py, uint32_t tile[kPatchLen][kPatchLen])
{
    for (int r = 0; r < kPatchLen; ++r)
        for (int c = 0; c < kPatchLen; ++c) tile[r][c] = 0;
    const int cx0 = px * kPatchLen - (int)ps.ox, cy0 = py * kPatchLen - (int)ps.oy;
    pull_patch_classes(ps.list.data(), ps.prefix, 0, cx0, cy0, [&](int, bool mneg, bool tneg, int lo, int hi) {   // lane = column
        for (int lane = 0; lane < kPatchLen; ++lane) {
            const int m = cx0 + lane;
            if (m == 0 || (m < 0) != mneg) continue;
            for (int i = lo; i < hi; ++i) {
                const int pos = pull_land(ps.list[i], (uint32_t)(m < 0 ? -m : m), tneg, cy0);
                if (pos >= 0) ++tile[pos][lane];
            }
        }
    });
    pull_patch_classes(ps.list.data(), ps.prefix, 4, cy0, cx0, [&](int, bool mneg, bool tneg, int lo, int hi) {   // lane = row
        for (int lane = 0; lane < kPatchLen; ++lane) {
            const int m = cy0 + lane;
            if (m == 0 || (m < 0) != mneg) continue;
            for (int i = lo; i < hi; ++i) {
                const int pos = pull_land(ps.list[i], (uint32_t)(m < 0 ? -m : m), tneg, cx0);
                if (pos >= 0) ++tile[lane][pos];
            }
        }
    });
}

bool update_maps_pull(Emu& e, const ScanParams& sp, const double* pts, const SE2& pose)
{
    const DirWindow win = e.occ.window;
    const uint32_t bx0 = (uint32_t)win.base_px << kPatchLog2, by0 = (uint32_t)win.base_py << kPatchLog2, side = (uint32_t)win.dim << kPatchLog2;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= win.dim) ++log2dim;
    Affine tf = compose_tf(pose, sp.moving);
    std::vector<uint32_t> tx(sp.n_beams), ty(sp.n_beams);
    std::vector<uint8_t> mh(sp.n_beams);
    uint32_t ox = 0, oy = 0;
    for (int b = 0; b < sp.n_beams; ++b) {
        const BeamCells bc = beam_cells(tf, sp, pts + 3 * b);
        const uint32_t fx = bc.from[0] - bx0, fy = bc.from[1] - by0;
        tx[b] = bc.to[0] - bx0; ty[b] = bc.to[1] - by0;
        mh[b] = bc.mark_hit;
        if (bc.from[2] != bc.to[2] || (fx | fy | tx[b] | ty[b]) >= side) return false;   // not planar / outside the window: the per-beam walk handles it
        if (b == 0) { ox = fx; oy = fy; }
        else if (fx != ox || fy != oy) return false;                                      // no common origin (truncated rays)
    }
    PullScan ps;
    pull_setup(ps, ox, oy, tx, ty, mh, win.dim);
    std::vector<uint64_t> events;
    uint32_t n_cand_touch = 0;
    static uint32_t tile[kPatchLen][kPatchLen];
    for (int py = 0; py < win.dim; ++py)
        for (int px = 0; px < win.dim; ++px) {
            const uint32_t di = ((uint32_t)py << log2dim) | (uint32_t)px;
            if (!ps.marked[di]) continue;
            pull_patch_counts(ps, px, py, tile);
            const int h_lo = ps.hit_lo[di], h_hi = h_lo + ps.hit_n[di];
            for (int r = 0; r < kPatchLen; ++r)
                for (int c = 0; c < kPatchLen; ++c) {
                    const uint32_t x = bx0 + (uint32_t)(px * kPatchLen + c), y = by0 + (uint32_t)(py * kPatchLen + r);
                    const uint32_t ci = cell_index(x, y);
                    int n_hit = 0;
                    for (int i = h_lo; i < h_hi; ++i) n_hit += pull_hit_cell(ps.hits[i]) == ci;
                    const uint32_t cnt = tile[r][c];
                    if (cnt == 0 && n_hit == 0) continue;   // untouched: the patch is not even allocated for it
                    uint32_t* cell = e.occ.raw(x, y, true);
                    uint8_t& fb = e.occ.fbit[cell - e.occ.cells.data()];
                    if (!fb && n_hit == 0) {   // plain cell: counter additions commute
                        *cell += cnt * kOccMissInc;
                        continue;
                    }
                    const PullRuns runs = pull_cell_runs(ps.list.data(), ps.prefix, px * kPatchLen + c - (int)ps.ox, py * kPatchLen + r - (int)ps.oy);
                    bool obstacle = fb != 0;
                    const uint32_t key = cell_key(win, x, y);
                    const uint32_t before = *cell;
                    *cell = pull_replay_cell(ps.list.data(), runs, ps.hits.data(), h_lo, h_hi, ci, before, obstacle,
                                             [&](bool add, uint32_t seq) { events.push_back(push_record((seq << 1) | (add ? 1u : 0u), key)); });
                    // the replay must have consumed exactly the counted crossings and the hits
                    if (*cell != before + cnt * kOccMissInc + (uint32_t)n_hit * kOccHitInc) e.occ.err |= 0x100u;
                    fb = obstacle;
                    n_cand_touch += cnt + (uint32_t)n_hit;
                }
        }
    run_brushfire(e, events, ps.cells, n_cand_touch);
    return true;
}

ScanParams scan_params(const Emu& e, int n)
{
    ScanParams sp{};
    sp.n_beams = n;
    sp.scale = e.scale;
    for (int i = 0; i < 9; ++i) sp.moving.l[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return sp;
}
}  // namespace

extern "C" {

// random push/pop sequence against std::priority_queue with the reference's comparator; returns #mismatches
int emu_heap_check(uint32_t seed, int n_ops, int prio_range)
{
    struct Cmp { bool operator()(const std::pair<int, uint32_t>& l, const std::pair<int, uint32_t>& r) const { return l.first > r.first; } };
    std::priority_queue<std::pair<int, uint32_t>, std::vector<std::pair<int, uint32_t>>, Cmp> ref;
    std::vector<uint64_t> buf(n_ops + 1);
    Heap h{buf.data(), 0u, (uint32_t)buf.size()};
    std::mt19937 g(seed);
    int bad = 0;
    uint32_t id = 0;
    for (int i = 0; i < n_ops; ++i) {
        if (h.size == 0 || (g() % 100) < 58) {
            int p = (int)(g() % prio_range);
            ref.push({p, id});
            heap_push(h, heap_entry((uint32_t)p, id));
            ++id;
        } else {
            auto t = ref.top();
            ref.pop();
            uint64_t e = heap_pop(h);
            if ((int)heap_prio(e) != t.first || heap_key(e) != t.second) ++bad;
        }
        if (h.size != ref.size()) ++bad;
    }
    while (!ref.empty()) {
        auto t = ref.top();
        ref.pop();
        uint64_t e = heap_pop(h);
        if ((int)heap_prio(e) != t.first || heap_key(e) != t.second) ++bad;
    }
    return bad;
}

// packed-cell helpers of the ray-cast kernel against the plain addressing functions, for every cell of a dim x dim window
int emu_packed_cell_check(int log2dim)
{
    DirWindow w;
    w.dim = 1 << log2dim; w.base_px = 1000; w.base_py = 2000;
    int bad = 0;
    const uint32_t side = (uint32_t)w.dim << kPatchLog2;
    for (uint32_t y = 0; y < side; ++y)
        for (uint32_t x = 0; x < side; ++x) {
            const uint32_t P = (y << 16) | x, ax = x + ((uint32_t)w.base_px << kPatchLog2), ay = y + ((uint32_t)w.base_py << kPatchLog2);
            if ((int)packed_dir_index(P, log2dim) != dir_index(w, ax, ay) || packed_cell_offset(P) != 4u * cell_index(ax, ay) || P != cell_key(w, ax, ay)) ++bad;
        }
    return bad;
}

// SegWalk (the ray-cast kernel's planar walk: packed cell, major/minor state, closed-form start at any step) against the
// reference's iterative walk (RayWalk = Map::computeRay, itself checked against the oracle by the SLAM emulation).  The beam is
// cut into segments of `seg` steps like the kernel's work items; every beam from the centre to every cell of a (2 r + 1)^2
// square when r > 0, else `count` random beams inside a window of `side` cells.  Returns the number of beams that differ.
int emu_segwalk_check(int r, uint32_t seed, int count, int side, int seg)
{
    int bad = 0;
    auto one = [&](uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty) {
        BeamCells bc;
        bc.from[0] = fx; bc.from[1] = fy; bc.from[2] = 7u;
        bc.to[0] = tx; bc.to[1] = ty; bc.to[2] = 7u;
        bc.mark_hit = true;
        RayWalk ref(bc);
        const int n = ref.n;
        bool ok = true;
        int i = 0;
        for (int s0 = 0; s0 == 0 || s0 < n - 1; s0 += seg) {
            SegWalk w;
            w.init(fx, fy, tx, ty, s0, seg);
            if (s0 == 0) {   // the first segment of a group is walked with next() (run merging)
                while (w.next()) ok = ok && ref.next() && w.i == ++i && (w.P & 0xFFFFu) == ref.x && (w.P >> 16) == ref.y;
            } else {         // the other segments with the kernel's counter-driven loop: one step ahead of the cell being processed, no end test in the walk
                int rem = w.iend - w.i;
                if (rem > 0) {
                    w.step();
                    uint32_t P = w.P;
                    for (;;) {
                        const int pos = w.i;
                        w.step();   // may land one cell past the segment (at most the beam's end cell): never processed
                        const uint32_t Pn = w.P;
                        ok = ok && ref.next() && pos == ++i && (P & 0xFFFFu) == ref.x && (P >> 16) == ref.y;
                        if (--rem == 0) break;
                        P = Pn;
                    }
                    // the look-ahead cell stays inside the bounding box of the beam's end cells
                    const uint32_t lx = w.P & 0xFFFFu, ly = w.P >> 16;
                    ok = ok && lx >= (fx < tx ? fx : tx) && lx <= (fx < tx ? tx : fx) && ly >= (fy < ty ? fy : ty) && ly <= (fy < ty ? ty : fy);
                }
            }
        }
        if (ref.next()) ok = false;   // the segments must cover every interior cell
        if (!ok) ++bad;
    };
    if (r > 0) {
        for (int ty = -r; ty <= r; ++ty)
            for (int tx = -r; tx <= r; ++tx) one(2000u, 2000u, (uint32_t)(2000 + tx), (uint32_t)(2000 + ty));
    } else {
        std::mt19937 g(seed);
        for (int c = 0; c < count; ++c) one(g() % side, g() % side, g() % side, g() % side);
    }
    return bad;
}

// ldlt_solve3 (named scalars, compile-time indices: what k_match runs) against ldlt_solve3_indexed (the original run-time indexed formulation): the same
// bits for random symmetric matrices of every kind the solver can meet -- positive definite, indefinite, rank deficient, equal diagonal entries (pivot ties),
// zeros.  Returns the number of systems whose three solution components are not bit-identical.
int emu_ldlt_check(uint32_t seed, int count)
{
    std::mt19937_64 g(seed);
    std::uniform_real_distribution<double> u(-1.0, 1.0);
    int bad = 0;
    for (int c = 0; c < count; ++c) {
        double a[6], b[3], h1[3], h2[3];
        const int kind = c % 8;
        double J[3][3];
        for (auto& r : J) for (double& v : r) v = u(g) * (kind == 1 ? 1e3 : 1.0);
        if (kind <= 2) {            // J^T J: positive semi-definite like the normal equations
            if (kind == 2) for (int j = 0; j < 3; ++j) J[2][j] = J[0][j] + J[1][j];   // rank 2
            int q = 0;
            for (int i = 0; i < 3; ++i)
                for (int j = i; j < 3; ++j) { double v = 0; for (int k = 0; k < 3; ++k) v += J[k][i] * J[k][j]; a[q++] = v; }
        } else {
            for (double& v : a) v = u(g);
            if (kind == 4) a[3] = a[0];                    // pivot ties on the diagonal
            if (kind == 5) { a[3] = a[0]; a[5] = a[0]; }
            if (kind == 6) { a[0] = 0.0; a[1] = 0.0; a[2] = 0.0; }   // a zero row / column
            if (kind == 7) for (double& v : a) v = 0.0;    // everything zero
        }
        for (double& v : b) v = u(g);
        lama_b200::ldlt_solve3(a, b, h1);
        lama_b200::ldlt_solve3_indexed(a, b, h2);
        if (std::memcmp(h1, h2, sizeof(h1)) != 0) ++bad;
    }
    return bad;
}

// one solve of k_match's 3x3 system A h = b (A by its upper triangle {A00,A01,A02,A11,A12,A22})
void emu_ldlt_solve(const double* a, const double* b, double* h) { lama_b200::ldlt_solve3(a, b, h); }
// Loc2D's covariance from the sums of the final evaluation (sums[0..5] = J^T J) of a scan of `rows` beams
void emu_covariance(const double* sums, uint64_t rows, double* cov) { lama_b200::covariance_from_sums(sums, (size_t)rows, cov); }

// ray_pull.h against the iterative walk: random beam sets from one origin inside a window of dim x dim patches.
//   mode 0: scan-like fan (even angles, noisy ranges)   1: random end cells   2: short beams (n = 0, 1, 2, ...)   3: axes / diagonals
// Checks (a) the marked patches cover every touched cell, (b) the chained counts of every cell of every marked patch, (c) for
// every touched cell the runs enumerate exactly the crossing beams with their step index, in beam order through pull_next_touch.
// Returns the number of mismatches.
int emu_pull_check(uint32_t seed, int n_beams, int mode, int dim)
{
    std::mt19937 g(seed);
    const int side = dim * kPatchLen;
    int log2dim = 0;
    while ((1 << (log2dim + 1)) <= dim) ++log2dim;
    const uint32_t ox = (uint32_t)(side / 4 + (int)(g() % (uint32_t)(side / 2))), oy = (uint32_t)(side / 4 + (int)(g() % (uint32_t)(side / 2)));
    std::vector<uint32_t> tx(n_beams), ty(n_beams);
    std::vector<uint8_t> mh(n_beams, 1);
    auto clampc = [&](int v) { return (uint32_t)std::min(std::max(v, 0), side - 1); };
    for (int b = 0; b < n_beams; ++b) {
        int x, y;
        if (mode == 0) {
            const double ang = -2.356 + 4.712 * b / std::max(1, n_beams - 1) + 1e-3 * (double)(g() % 100);
            const double r = 4.0 + (double)(g() % (uint32_t)(side / 2));
            x = (int)ox + (int)std::lround(r * std::cos(ang)); y = (int)oy + (int)std::lround(r * std::sin(ang));
        } else if (mode == 1) {
            x = (int)(g() % (uint32_t)side); y = (int)(g() % (uint32_t)side);
        } else if (mode == 2) {
            x = (int)ox + (int)(g() % 9) - 4; y = (int)oy + (int)(g() % 9) - 4;
        } else {
            const int r = (int)(g() % (uint32_t)(side / 3)), k = (int)(g() % 8);
            const int dx[8] = {1, 1, 0, -1, -1, -1, 0, 1}, dy[8] = {0, 1, 1, 1, 0, -1, -1, -1};
            x = (int)ox + r * dx[k] + ((g() % 4) == 0 ? (int)(g() % 3) - 1 : 0); y = (int)oy + r * dy[k] + ((g() % 4) == 0 ? (int)(g() % 3) - 1 : 0);
        }
        tx[b] = clampc(x); ty[b] = clampc(y);
        mh[b] = (g() % 8) != 0;
    }
    // brute force
    std::vector<uint32_t> ref((size_t)side * side, 0u);
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> who((size_t)side * side);   // (beam, step)
    uint32_t ref_cells = 0;
    for (int b = 0; b < n_beams; ++b) {
        BeamCells bc;
        bc.from[0] = ox; bc.from[1] = oy; bc.from[2] = 5u; bc.to[0] = tx[b]; bc.to[1] = ty[b]; bc.to[2] = 5u; bc.mark_hit = mh[b];
        RayWalk w(bc);
        uint32_t step = 0;
        ref_cells += mh[b] ? 1u : 0u;
        while (w.next()) {
            ++step; ++ref_cells;
            ++ref[(size_t)w.y * side + w.x];
            who[(size_t)w.y * side + w.x].push_back({(uint32_t)b, step});
        }
    }
    PullScan ps;
    pull_setup(ps, ox, oy, tx, ty, mh, dim);
    int bad = 0;
    if (ps.cells != ref_cells) ++bad;
    // slope order inside the classes must be the exact rational order
    for (int c = 0; c < 8; ++c)
        for (int i = ps.prefix[c] + 1; i < ps.prefix[c + 1]; ++i) {
            const uint64_t n0 = ps.list[i - 1].nd & 0xFFFFu, d0 = ps.list[i - 1].nd >> 16, n1 = ps.list[i].nd & 0xFFFFu, d1 = ps.list[i].nd >> 16;
            if (d0 * n1 > d1 * n0) ++bad;
        }
    static uint32_t tile[kPatchLen][kPatchLen];
    for (int py = 0; py < dim; ++py)
        for (int px = 0; px < dim; ++px) {
            const bool marked = ps.marked[((size_t)py << log2dim) | (size_t)px] != 0;
            if (marked) {
                pull_patch_counts(ps, px, py, tile);
            }
            for (int r = 0; r < kPatchLen; ++r)
                for (int c = 0; c < kPatchLen; ++c) {
                    const int x = px * kPatchLen + c, y = py * kPatchLen + r;
                    const uint32_t want = ref[(size_t)y * side + x];
                    if (!marked) {
                        if (want) ++bad;
                        continue;
                    }
                    if (tile[r][c] != want) ++bad;
                    if (!want) continue;
                    const PullRuns runs = pull_cell_runs(ps.list.data(), ps.prefix, x - (int)ox, y - (int)oy);
                    std::vector<std::pair<uint32_t, uint32_t>> got;
                    int after = -1;
                    for (;;) {
                        const PullTouch t = pull_next_touch(ps.list.data(), runs, pull_cell_hits(ps.hits.data(), 0, 0, 0u), ps.hits.data(), 0, 0, 0u, after);
                        if (!t.valid) break;
                        got.push_back({t.beam, t.pos});
                        after = (int)t.beam;
                    }
                    auto w = who[(size_t)y * side + x];
                    std::sort(w.begin(), w.end());
                    if (got != w) ++bad;
                }
        }
    return bad;
}
// pull_minor_at (division by 2 n as a multiplication) against the plain division: every n, d <= n, and the a around every jump of k
int emu_magic_check(int n_max)
{
    int bad = 0;
    for (uint32_t n = 1; n <= (uint32_t)n_max; ++n) {
        const uint64_t magic = pull_magic(n);
        // all dividends x = 2 a d + n with a, d < 4096 are below 2^25: check the floor at every multiple of 2 n in that range, just below and at it
        for (uint64_t q = 0; q * 2 * n < (1ull << 25); ++q) {
            const uint64_t x1 = q * 2 * n, x0 = x1 ? x1 - 1 : 0, x2 = x1 + 2 * n - 1;
            if (((x1 * magic) >> 38) != x1 / (2 * n) || ((x0 * magic) >> 38) != x0 / (2 * n)) ++bad;
            if (x2 < (1ull << 25) && ((x2 * magic) >> 38) != x2 / (2 * n)) ++bad;
        }
        const uint32_t ds[4] = {0u, 1u, n / 2, n};
        for (uint32_t d : ds)
            for (uint32_t a = 1; a < 4096; a += (a < 64 ? 1 : 37))
                if (pull_minor_at(pull_pack(n, d), magic, a) != (2u * a * d + n) / (2u * n)) ++bad;
    }
    return bad;
}
void emu_set_pull(void* h, int on) { ((Emu*)h)->pull = on != 0; }
uint32_t emu_pull_fallbacks(void* h) { return ((Emu*)h)->pull_fallbacks; }

void* emu_create(double resolution, double l2_max, double cx, double cy, int dir_dim, double trans_thresh, double rot_thresh, uint32_t max_iter, int strategy)
{
    Emu* e = new Emu();
    e->resolution = resolution;
    e->scale = 1.0 / resolution;
    uint32_t r = (uint32_t)std::ceil(l2_max * e->scale);
    e->max_sqdist = r * r;
    DirWindow w;
    w.dim = dir_dim;
    w.base_px = (int32_t)(w2m(cx, e->scale) >> kPatchLog2) - dir_dim / 2;
    w.base_py = (int32_t)(w2m(cy, e->scale) >> kPatchLog2) - dir_dim / 2;
    e->occ.init(w);
    e->dm.init(w);
    e->trans_thresh = trans_thresh;
    e->rot_thresh = rot_thresh;
    e->max_iter = max_iter;
    e->strategy = strategy;
    return e;
}
void emu_destroy(void* h) { delete (Emu*)h; }
void emu_set_pose(void* h, double x, double y, double r) { ((Emu*)h)->pose = se2_from_xyr(x, y, r); }
void emu_get_state(void* h, double* s) { Emu* e = (Emu*)h; s[0] = e->pose.c; s[1] = e->pose.s; s[2] = e->pose.tx; s[3] = e->pose.ty; }
void emu_counters(void* h, uint32_t* c) { Emu* e = (Emu*)h; c[0] = e->last_evals; c[1] = e->last_cells; c[2] = e->last_pops; c[3] = e->last_events; c[4] = e->last_log; c[5] = e->last_iters; c[6] = e->occ.err | e->dm.err; }

// Slam2D::update (src/slam2d.cpp:143-198) on top of the emulated kernels
int emu_slam_update(void* h, const double* pts, int n, const double* odom_xyr, uint32_t shuffle_seed)
{
    Emu* e = (Emu*)h;
    ScanParams sp = scan_params(*e, n);
    const SE2 odometry = se2_from_xyr(odom_xyr[0], odom_xyr[1], odom_xyr[2]);
    if (!e->has_first) {
        e->odom = odometry;
        update_maps(*e, sp, pts, e->pose, shuffle_seed);
        e->has_first = true;
        return 1;
    }
    const SE2 odelta = se2_mul(se2_inv(e->odom), odometry);
    const SE2 ppose = se2_mul(e->pose, odelta);
    if (std::sqrt(odelta.tx * odelta.tx + odelta.ty * odelta.ty) <= e->trans_thresh && std::fabs(se2_rotation(odelta)) <= e->rot_thresh) return 0;
    e->pose = ppose;
    e->odom = odometry;
    SolverOptions so{};
    so.strategy = e->strategy; so.robust_kind = kRobustCauchy; so.robust_param = 0.15; so.max_iterations = e->max_iter;
    so.eps1 = so.eps2 = so.tau = 1e-4;
    double sums[kNumSums];
    solve(*e, sp, pts, e->pose, so, sums);
    update_maps(*e, sp, pts, e->pose, shuffle_seed);
    return 1;
}

void emu_export_dm(void* h, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy, uint8_t* queued)
{
    Emu* e = (Emu*)h;
    for (int j = 0; j < hh; ++j)
        for (int i = 0; i < w; ++i) {
            uint32_t x = x0 + i, y = y0 + j;
            uint32_t d = dir_index(e->dm.window, x, y) < 0 ? 0u : *e->dm.raw(x, y, false);
            uint32_t o = dir_index(e->occ.window, x, y) < 0 ? 0u : *e->occ.raw(x, y, false);
            int k = j * w + i;
            sqdist[k] = (uint16_t)dm_sqdist(d); valid[k] = (d & kDmValid) != 0; ox[k] = (int16_t)dm_ox(d); oy[k] = (int16_t)dm_oy(d);
            queued[k] = (d & kDmQueued) != 0;
            known[k] = (d & kDmKnown) != 0 || o != 0;
        }
}
void emu_export_occ(void* h, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* occupied, uint16_t* visited, uint8_t* obstacle)
{
    Emu* e = (Emu*)h;
    for (int j = 0; j < hh; ++j)
        for (int i = 0; i < w; ++i) {
            uint32_t x = x0 + i, y = y0 + j;
            const bool in = dir_index(e->occ.window, x, y) >= 0;
            uint32_t* c = in ? e->occ.raw(x, y, false) : nullptr;
            uint32_t o = in ? *c : 0u;
            int k = j * w + i;
            occupied[k] = (uint16_t)occ_occupied(o); visited[k] = (uint16_t)occ_visited(o); obstacle[k] = in ? e->occ.fbit[c - e->occ.cells.data()] : 0;
        }
}
// direct brushfire calls for the stand-alone DDM comparison
uint32_t emu_dm_apply(void* h, const uint32_t* cells_xy, const uint8_t* is_add, int n)
{
    Emu* e = (Emu*)h;
    e->heap_l.assign(1 << 16, 0);
    e->heap_r.assign(1 << 16, 0);
    Brushfire<HostDm> bf(e->dm, Heap{e->heap_r.data(), 0u, (uint32_t)e->heap_r.size()}, Heap{e->heap_l.data(), 0u, (uint32_t)e->heap_l.size()}, e->max_sqdist);
    for (int i = 0; i < n; ++i) {
        if (is_add[i]) bf.add_obstacle(cells_xy[2 * i], cells_xy[2 * i + 1]);
        else bf.remove_obstacle(cells_xy[2 * i], cells_xy[2 * i + 1]);
    }
    const uint32_t pops = bf.update();
    note_heap_peak(*e, bf);
    return pops;
}
// largest lower [0] and raise [1] heap size of any brushfire of this emulation so far (k_brushfire keeps the first
// BrushParams::lower_cap / raise_cap entries in shared memory)
void emu_heap_peak(void* h, uint32_t* out)
{
    Emu* e = (Emu*)h;
    out[0] = e->heap_peak[0];
    out[1] = e->heap_peak[1];
}
// replay_cell (ray_core.h) on one frequency cell as k_raycast runs it: the touches kinds[i] (1 hit / 0 miss, beam order) are first
// added to the packed word {visited, occupied} = word_in (packed adds carry from occupied into visited; they commute, so their
// order does not matter), then replayed; returns the word the replay stores.  events_out[i] = 1 add, 2 remove, 0 none
uint32_t emu_freq_replay(const uint8_t* kinds, int n, uint32_t word_in, int obstacle_in, uint8_t* events_out, int* obstacle_out)
{
    std::vector<uint64_t> log((size_t)n);
    uint32_t word = word_in;
    for (int i = 0; i < n; ++i) {
        word += kinds[i] ? kOccHitInc : kOccMissInc;
        log[i] = log_record(7u, (uint32_t)i, kinds[i] ? 0u : 1u, kinds[i] != 0);
        events_out[i] = 0;
    }
    const bool obstacle = replay_cell(log.data(), 0, n, word, obstacle_in != 0, [&](bool add, uint32_t seq) { events_out[seq >> 15] = add ? 1 : 2; });
    *obstacle_out = obstacle;
    return word;
}
// replay_cell_prob (ray_core.h) on one cell: kinds[i] = 1 hit / 0 miss in beam order; events_out[i] = 1 add, 2 remove, 0 none
float emu_prob_replay(const uint8_t* kinds, int n, const double* constants, int obstacle_in, uint8_t* events_out, int* obstacle_out)
{
    std::vector<uint64_t> log((size_t)n);
    for (int i = 0; i < n; ++i) {
        log[i] = log_record(7u, (uint32_t)i, kinds[i] ? 0u : 1u, kinds[i] != 0);
        events_out[i] = 0;
    }
    ProbParams pp{constants[0], constants[1], constants[2], constants[3], constants[4]};
    bool obstacle = obstacle_in != 0;
    float p = replay_cell_prob(log.data(), 0, n, 0.0f, obstacle, pp, [&](bool add, uint32_t seq) { events_out[seq >> 15] = add ? 1 : 2; });
    *obstacle_out = obstacle;
    return p;
}
// SE2 helpers of lama_core.h for comparison with the oracle's.  a is a state (c, s, tx, ty) for ops 0, 1 and 4 and a 3-vector for 2 and 3.
void emu_se2(int op, const double* a, const double* b, double* out)
{
    SE2 A{1, 0, 0, 0}, r{1, 0, 0, 0};
    if (op == 0 || op == 1 || op == 4) A = SE2{a[0], a[1], a[2], a[3]};
    if (op == 0) r = se2_mul(A, SE2{b[0], b[1], b[2], b[3]});
    else if (op == 1) r = se2_inv(A);
    else if (op == 2) r = se2_exp(a);
    else if (op == 3) r = se2_from_xyr(a[0], a[1], a[2]);
    else if (op == 4) { se2_log(A, out); out[3] = 0.0; return; }   // (upsilon, theta)
    out[0] = r.c; out[1] = r.s; out[2] = r.tx; out[3] = r.ty;
}
}
