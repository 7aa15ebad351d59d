// ddm3_core.h -- the dynamic brushfire of DynamicDistanceMap with is3d = true (six neighbours), executed as ONE logical sequential
// thread per map, bit-faithful to a libstdc++ build of the reference:
//   src/sdm/dynamic_distance_map.cpp:160-197 (update), :212-242 (add/removeObstacle), :244-279 (raise), :281-330 (lower),
//   neighbour order :40-45.
//
// Parity needs the exact std::priority_queue pop order (DESIGN.md §5, §12), so the heaps are ddm_core.h's Heap / heap_push /
// heap_pop, unchanged, with entries prio << 32 | key and key = directory entry << 15 | cell index (a window has at most 65 536
// entries, so the key fits 31 bits).
//
// The code is written against a `Map` policy so that the same source runs inside k_dm3_brushfire (ddm3d.cu) against the device
// pool and on the host in tests/emu/ddm3_emu.cpp:
//   uint64_t* cell(x, y, z)  -- the MUTABLE Map::get (map.cpp:371-412): allocates the patch on first touch, marks the cell known,
//                               never returns null (an out-of-window or out-of-pool access returns a scratch cell and raises an
//                               error bit)
//   PatchWindow win
//
// Memory safety rests on a host-side admission (Dm3Guard below) that both the device map and the emulation apply before any write:
// with R = ceil(l2_max * scale), every cell the brushfire touches lies within R cells, on every axis, of a cell of an admitted batch
// (or of the obstacle of a valid cell read from a file), because a valid cell is less than R from its obstacle on every axis.
#pragma once

#include <string>
#include <vector>

#include "ddm_core.h"
#include "patch_window.h"
#include "trilinear.h"

namespace lama_b200 {

// ---- cell ------------------------------------------------------------------------------------------------------------------------
// One 8-byte word per cell, the little-endian image of
//   struct { int8 ox, oy, oz; uint8 flags; uint16 sqdist; uint16 unused; }
// flags: kDm3Valid (valid_obstacle), kDm3Queued (is_queued), kDm3Known (the Container mask bit).  The reference's int16 offsets fit 8
// bits because a valid cell has |offset|^2 = sqdist < max_sqdist <= 63^2.  A patch is 32^3 cells, 256 KiB.
constexpr int kDm3Log2Cells    = 3 * kPatchLog2;
constexpr int kDm3Cells        = 1 << kDm3Log2Cells;
constexpr int kDm3MaxEntries   = 1 << 16;
constexpr uint32_t kDm3Valid   = 1u;
constexpr uint32_t kDm3Queued  = 2u;
constexpr uint32_t kDm3Known   = 4u;
constexpr int kDm3FlagShift    = 24;
constexpr int kDm3SqShift      = 32;
constexpr uint32_t kDm3HeapRoom = 6;   // the pushes one pop can make

LAMA_HD int dm3_off(uint64_t c, int k) { return (int)(int8_t)(uint8_t)(c >> (8 * k)); }
LAMA_HD uint32_t dm3_flags(uint64_t c) { return (uint32_t)(c >> kDm3FlagShift) & 0xFFu; }
LAMA_HD uint32_t dm3_sqdist(uint64_t c) { return (uint32_t)(c >> kDm3SqShift) & 0xFFFFu; }
LAMA_HD bool dm3_valid(uint64_t c) { return (dm3_flags(c) & kDm3Valid) != 0; }
LAMA_HD bool dm3_queued(uint64_t c) { return (dm3_flags(c) & kDm3Queued) != 0; }
LAMA_HD bool dm3_known(uint64_t c) { return (dm3_flags(c) & kDm3Known) != 0; }
LAMA_HD uint64_t dm3_pack(uint32_t sqdist, int ox, int oy, int oz, bool valid, bool queued)
{
    const uint32_t fl = kDm3Known | (valid ? kDm3Valid : 0u) | (queued ? kDm3Queued : 0u);
    return (uint64_t)(uint8_t)ox | ((uint64_t)(uint8_t)oy << 8) | ((uint64_t)(uint8_t)oz << 16) | ((uint64_t)fl << kDm3FlagShift) |
           ((uint64_t)(sqdist & 0xFFFFu) << kDm3SqShift);
}
constexpr uint64_t kDm3QueuedBit = (uint64_t)kDm3Queued << kDm3FlagShift;
constexpr uint64_t kDm3KnownBit  = (uint64_t)kDm3Known << kDm3FlagShift;

LAMA_HD uint32_t dm3_cell_index(uint32_t x, uint32_t y, uint32_t z) { return window_cell_index(x, y, z, 1); }
// heap key -> cell
LAMA_HD void dm3_key_cell(const PatchWindow& w, uint32_t key, uint32_t& x, uint32_t& y, uint32_t& z)
{
    uint32_t a[3];
    window_anchor(w, (int)(key >> kDm3Log2Cells), a);
    const uint32_t ci = key & (uint32_t)(kDm3Cells - 1);
    x = a[0] | (ci & (kPatchLen - 1));
    y = a[1] | ((ci >> kPatchLog2) & (kPatchLen - 1));
    z = a[2] | (ci >> (2 * kPatchLog2));
}

// ---- resumable run ---------------------------------------------------------------------------------------------------------------
// What a run leaves for the next one: it lives in device memory between launches of k_dm3_brushfire.
enum : uint32_t { kDm3Done = 0, kDm3NeedRoom = 1, kDm3Budget = 2 };
struct Dm3State {
    uint32_t raise_size, lower_size;   // heap entries
    uint32_t next_op;                  // pending add / remove ops applied so far
    uint32_t processed;                // update()'s count so far
    uint32_t used;                     // pool slots taken
    uint32_t err;                      // kErr* bits (lama_core.h); never set when the host admission holds
    uint32_t stop;                     // how the last run ended: kDm3Done, kDm3NeedRoom (a heap lacks room), kDm3Budget (pop budget spent)
    uint32_t seg;                      // run_segments: segments finished so far
};
// a pending op: x, y, z, kind (0 addObstacle, 1 removeObstacle)
constexpr int kDm3OpWords = 4;

template <typename Map>
struct Brushfire3 {
    Map& map;
    Heap raise_q, lower_q;
    uint32_t max_sqdist;
    uint32_t err = 0;

    LAMA_HD Brushfire3(Map& m, Heap r, Heap l, uint32_t msq) : map(m), raise_q(r), lower_q(l), max_sqdist(msq) {}

    LAMA_HD void push(Heap& q, uint32_t prio, uint32_t x, uint32_t y, uint32_t z)
    {
        const int di = window_dir_index(map.win, x, y, z);
        if (di < 0) { err |= kErrWindow; return; }
        if (!heap_push(q, heap_entry(prio, ((uint32_t)di << kDm3Log2Cells) | dm3_cell_index(x, y, z)))) err |= kErrHeapOverflow;
    }

    // dynamic_distance_map.cpp:212-226
    LAMA_HD void add_obstacle(uint32_t x, uint32_t y, uint32_t z)
    {
        uint64_t* c = map.cell(x, y, z);
        const uint64_t w = *c;
        if (dm3_valid(w) && dm3_sqdist(w) == 0) return;
        *c = dm3_pack(0, 0, 0, 0, true, true);
        push(lower_q, 0, x, y, z);
    }
    // :228-242
    LAMA_HD void remove_obstacle(uint32_t x, uint32_t y, uint32_t z)
    {
        uint64_t* c = map.cell(x, y, z);
        const uint64_t w = *c;
        if (!(dm3_valid(w) && dm3_sqdist(w) == 0)) return;
        *c = dm3_pack(0, 0, 0, 0, false, true);
        push(raise_q, 0, x, y, z);
    }

    // :244-279 ; neighbour order (+1,0,0) (0,+1,0) (-1,0,0) (0,-1,0) (0,0,+1) (0,0,-1) (:40-45)
    LAMA_HD void raise(uint32_t x, uint32_t y, uint32_t z, uint64_t* cur)
    {
        const int dx[6] = {1, 0, -1, 0, 0, 0}, dy[6] = {0, 1, 0, -1, 0, 0}, dz[6] = {0, 0, 0, 0, 1, -1};
        for (int i = 0; i < 6; ++i) {
            const uint32_t nx = x + dx[i], ny = y + dy[i], nz = z + dz[i];
            uint64_t* nb = map.cell(nx, ny, nz);
            const uint64_t n = *nb;
            if (dm3_queued(n) || !dm3_valid(n)) continue;
            const uint64_t o = *map.cell(nx + dm3_off(n, 0), ny + dm3_off(n, 1), nz + dm3_off(n, 2));
            if (!dm3_valid(o)) {
                push(raise_q, dm3_sqdist(n), nx, ny, nz);
                *nb = dm3_pack(0, 0, 0, 0, false, true);
            } else {   // `else if (not neighbor->is_queued)` is always taken here
                push(lower_q, dm3_sqdist(n), nx, ny, nz);
                *nb = n | kDm3QueuedBit;
            }
        }
        *cur &= ~kDm3QueuedBit;
    }

    // :281-330
    LAMA_HD void lower(uint32_t x, uint32_t y, uint32_t z, uint64_t* cur)
    {
        const uint64_t c = *cur;
        if (!dm3_queued(c)) return;
        const int co[3] = {dm3_off(c, 0), dm3_off(c, 1), dm3_off(c, 2)};
        const int dx[6] = {1, 0, -1, 0, 0, 0}, dy[6] = {0, 1, 0, -1, 0, 0}, dz[6] = {0, 0, 0, 0, 1, -1};
        for (int i = 0; i < 6; ++i) {
            if (dx[i] * co[0] > 0 || dy[i] * co[1] > 0 || dz[i] * co[2] > 0) continue;   // only update away from the obstacle (:296)
            const uint32_t nx = x + dx[i], ny = y + dy[i], nz = z + dz[i];
            uint64_t* nb = map.cell(nx, ny, nz);
            const uint64_t n = *nb;
            // the current cell's obstacle, relative to the neighbour
            const int rx = co[0] - dx[i], ry = co[1] - dy[i], rz = co[2] - dz[i];
            const uint32_t new_sq = (uint32_t)(rx * rx + ry * ry + rz * rz);
            const uint32_t cmp_sq = dm3_valid(n) ? dm3_sqdist(n) : max_sqdist;
            bool overwrite = new_sq < cmp_sq;
            if (!overwrite && new_sq == dm3_sqdist(n)) {
                const uint64_t o = *map.cell(nx + dm3_off(n, 0), ny + dm3_off(n, 1), nz + dm3_off(n, 2));
                if (!dm3_valid(n) || !(dm3_valid(o) && dm3_sqdist(o) == 0)) overwrite = true;
            }
            if (overwrite) {
                push(lower_q, new_sq, nx, ny, nz);
                *nb = dm3_pack(new_sq, rx, ry, rz, true, true);
            }
        }
        *cur &= ~kDm3QueuedBit;
    }

    // Applies ops [s.next_op, n_ops) in list order, then (with do_update) runs update() (:160-197) from where s left it.  Stops at an
    // op or pop boundary when a heap lacks room for the pushes that step can make (kDm3NeedRoom) or after `budget` pops (kDm3Budget);
    // s then holds what the next run continues from.  The caller saves the heap sizes, the pool counter and err.
    LAMA_HD void run(Dm3State& s, const uint32_t* ops, uint32_t n_ops, bool do_update, uint64_t budget)
    {
        s.stop = kDm3Done;
        while (s.next_op < n_ops) {
            if (raise_q.size >= raise_q.cap || lower_q.size >= lower_q.cap) { s.stop = kDm3NeedRoom; return; }
            const uint32_t* o = ops + (size_t)kDm3OpWords * s.next_op;
            if (o[3]) remove_obstacle(o[0], o[1], o[2]);
            else add_obstacle(o[0], o[1], o[2]);
            ++s.next_op;
        }
        if (!do_update) return;
        for (uint64_t pops = 0;; ++pops) {
            const bool in_raise = raise_q.size != 0;
            if (!in_raise && lower_q.size == 0) return;
            if (raise_q.size + kDm3HeapRoom > raise_q.cap || lower_q.size + kDm3HeapRoom > lower_q.cap) { s.stop = kDm3NeedRoom; return; }
            if (pops >= budget) { s.stop = kDm3Budget; return; }
            uint32_t x, y, z;
            dm3_key_cell(map.win, heap_key(heap_pop(in_raise ? raise_q : lower_q)), x, y, z);
            uint64_t* cur = map.cell(x, y, z);
            ++s.processed;
            if (in_raise) {
                raise(x, y, z, cur);
                continue;
            }
            const uint64_t c = *cur;
            if (dm3_valid(c)) {
                const uint64_t o = *map.cell(x + dm3_off(c, 0), y + dm3_off(c, 1), z + dm3_off(c, 2));
                if (dm3_sqdist(o) == 0) lower(x, y, z, cur);
            }
        }
    }

    // The ops cut into n_seg segments, segment k ending at op seg_end[k]: from segment s.seg on, applies the segment's ops and runs
    // update() to the end, and writes its count to processed[k] (the reference's per-cloud update(), slam2d.cpp:271-316).  Stops and
    // resumes as run() does; `budget` bounds the pops of the whole call.
    LAMA_HD void run_segments(Dm3State& s, const uint32_t* ops, const uint32_t* seg_end, uint32_t n_seg, uint64_t budget, uint32_t* processed)
    {
        s.stop = kDm3Done;
        while (s.seg < n_seg) {
            const uint32_t p0 = s.processed;
            run(s, ops, seg_end[s.seg], true, budget);
            budget -= s.processed - p0;   // run() pops at most `budget`
            if (s.stop != kDm3Done) return;
            processed[s.seg] = s.processed;
            s.processed = 0;
            ++s.seg;
        }
    }
};

// at least `margin` cells inside the window on every axis
LAMA_HD bool dm3_inside(const PatchWindow& w, uint32_t x, uint32_t y, uint32_t z, int margin)
{
    const uint32_t c[3] = {x, y, z};
    for (int k = 0; k < 3; ++k) {
        const int64_t lo = ((int64_t)w.base[k] << kPatchLog2) + margin;
        const int64_t hi = (((int64_t)w.base[k] + w.dim[k]) << kPatchLog2) - 1 - margin;
        if ((int64_t)c[k] < lo || (int64_t)c[k] > hi) return false;
    }
    return true;
}

// ---- host admission --------------------------------------------------------------------------------------------------------------
// Decides, before anything is written, whether a batch of add / remove cells may enter the map.  `reachable` marks the directory
// entries within R cells (every axis) of a cell of an admitted batch or of a read file's obstacle: the only entries the brushfire can
// allocate.
struct Dm3Guard {
    PatchWindow win{};
    int reach = 0;                     // R = ceil(l2_max * scale), at most 63
    std::vector<uint8_t> reachable;    // per directory entry

    void init(const PatchWindow& w, int r)
    {
        win = w;
        reach = r;
        reachable.assign((size_t)w.dim[0] * w.dim[1] * w.dim[2], 0);
    }
    // at least R + 1 cells inside the window on every axis: then every cell within R of it is inside too
    bool inside(uint32_t x, uint32_t y, uint32_t z) const { return dm3_inside(win, x, y, z, reach + 1); }
    // marks in r the entries of the cells within R of (x, y, z), which must be inside()
    void mark(std::vector<uint8_t>& r, uint32_t x, uint32_t y, uint32_t z) const
    {
        const uint32_t R = (uint32_t)reach;
        for (uint32_t pz = (z - R) >> kPatchLog2; pz <= (z + R) >> kPatchLog2; ++pz)
            for (uint32_t py = (y - R) >> kPatchLog2; py <= (y + R) >> kPatchLog2; ++py)
                for (uint32_t px = (x - R) >> kPatchLog2; px <= (x + R) >> kPatchLog2; ++px)
                    r[(size_t)window_dir_index(win, px << kPatchLog2, py << kPatchLog2, pz << kPatchLog2)] = 1;
    }
    // marks in r the entries within R of any cell of entry di (those outside the window aside)
    void mark_entry(std::vector<uint8_t>& r, int di) const
    {
        uint32_t a[3];
        window_anchor(win, di, a);
        const uint32_t R = (uint32_t)reach;
        for (uint32_t pz = (a[2] - R) >> kPatchLog2; pz <= (a[2] + kPatchLen - 1 + R) >> kPatchLog2; ++pz)
            for (uint32_t py = (a[1] - R) >> kPatchLog2; py <= (a[1] + kPatchLen - 1 + R) >> kPatchLog2; ++py)
                for (uint32_t px = (a[0] - R) >> kPatchLog2; px <= (a[0] + kPatchLen - 1 + R) >> kPatchLog2; ++px) {
                    const int e = window_dir_index(win, px << kPatchLog2, py << kPatchLog2, pz << kPatchLog2);
                    if (e >= 0) r[(size_t)e] = 1;
                }
    }
    // The pool check of a batch that may add or remove obstacles anywhere in the marked entries (marks[i] != 0): -5 (pool) when the
    // reachable entries, with those within R of the marked ones, that have no patch could exceed free_slots; else 0 and next = them.
    // Nothing changes here: the caller commits next to `reachable` once the batch is admitted.
    int admit_entries(const std::vector<uint32_t>& marks, const std::vector<int32_t>& dir, int64_t free_slots, std::vector<uint8_t>& next,
                      std::string& err) const
    {
        next = reachable;
        for (size_t i = 0; i < marks.size(); ++i)
            if (marks[i]) mark_entry(next, (int)i);
        if (missing(next, dir) > free_slots) {
            err = "the distance-map patches this batch can reach could exceed the free pool slots (raise pool_slots)";
            return -5;
        }
        return 0;
    }
    // reachable entries of r without a patch in dir (-1 = none)
    static int64_t missing(const std::vector<uint8_t>& r, const std::vector<int32_t>& dir)
    {
        int64_t n = 0;
        for (size_t i = 0; i < r.size(); ++i) n += r[i] && dir[i] < 0;
        return n;
    }
    // LAMA status of admitting n cells (x, y, z triples at stride `stride` words) with free_slots pool slots left: -4 (window) when a
    // cell is less than R + 1 inside the window, -5 (pool) when the reachable entries without a patch could exceed the free slots, 0
    // after marking them.  Nothing changes on a refusal.
    int admit(const uint32_t* xyz, int64_t n, int stride, const std::vector<int32_t>& dir, int64_t free_slots, std::string& err)
    {
        for (int64_t i = 0; i < n; ++i) {
            const uint32_t* c = xyz + (size_t)stride * i;
            if (!inside(c[0], c[1], c[2])) {
                err = "cell " + std::to_string(i) + " lies less than " + std::to_string(reach + 1) + " cells (reach + 1) inside the directory window";
                return -4;
            }
        }
        std::vector<uint8_t> next = reachable;
        for (int64_t i = 0; i < n; ++i) {
            const uint32_t* c = xyz + (size_t)stride * i;
            mark(next, c[0], c[1], c[2]);
        }
        if (missing(next, dir) > free_slots) {
            err = "the patches this batch can reach could exceed the free pool slots (raise pool_slots)";
            return -5;
        }
        reachable.swap(next);
        return 0;
    }
};

}  // namespace lama_b200
