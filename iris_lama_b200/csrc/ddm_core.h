// ddm_core.h -- the dynamic brushfire of DynamicDistanceMap::update() executed as ONE logical
// sequential thread per particle, bit-faithful to a libstdc++ build of the reference:
//   src/sdm/dynamic_distance_map.cpp:160-197 (update), :212-242 (add/removeObstacle),
//   :244-279 (raise), :281-330 (lower); queue types include/lama/sdm/dynamic_distance_map.h:90-104.
//
// Why sequential: the result of the brushfire depends on the pop order of equal-priority heap
// entries (measured: thousands of differing cells under random tie orders on add/remove stress,
// see DESIGN.md), so parity with the reference requires the exact std::priority_queue order.  The
// binary-heap routines below reproduce libstdc++'s std::push_heap / std::pop_heap
// (bits/stl_heap.h: __push_heap, __adjust_heap) move for move; the comparator looks at the
// priority only, exactly like compare_prio.
//
// The code is written against a `Map` policy so that the same source runs (a) inside the CUDA
// kernel, warp-uniformly, against the device patch pool and (b) on the host in tests/emu.
#pragma once

#include "lama_core.h"

namespace lama_b200 {

// heap entry: priority in the high word, window-relative cell key in the low word
LAMA_HD uint64_t heap_entry(uint32_t prio, uint32_t key) { return ((uint64_t)prio << 32) | key; }
LAMA_HD uint32_t heap_prio(uint64_t e) { return (uint32_t)(e >> 32); }
LAMA_HD uint32_t heap_key(uint64_t e) { return (uint32_t)e; }
// compare_prio(left, right) == left.first > right.first
LAMA_HD bool heap_comp(uint64_t l, uint64_t r) { return heap_prio(l) > heap_prio(r); }

struct Heap {
    uint64_t* data;
    uint32_t size;
    uint32_t cap;
    uint32_t peak = 0;   // largest size reached (the host emulation reports it; the kernels use SmemHeap)
};

// std::push_heap after vector::push_back  (stl_heap.h __push_heap with topIndex = 0)
LAMA_HD bool heap_push(Heap& h, uint64_t value)
{
    if (h.size >= h.cap) return false;
    int64_t hole = h.size++;
    if (h.size > h.peak) h.peak = h.size;
    int64_t parent = (hole - 1) / 2;
    while (hole > 0 && heap_comp(h.data[parent], value)) {
        h.data[hole] = h.data[parent];
        hole         = parent;
        parent       = (hole - 1) / 2;
    }
    h.data[hole] = value;
    return true;
}

// std::pop_heap + vector::pop_back; returns the popped top  (stl_heap.h __pop_heap/__adjust_heap)
LAMA_HD uint64_t heap_pop(Heap& h)
{
    uint64_t top = h.data[0];
    uint32_t last = --h.size;           // element moved out of the back
    if (last == 0) return top;
    uint64_t value = h.data[last];
    const int64_t len = last;           // heap length after removing the back slot
    int64_t hole = 0, second = 0;
    while (second < (len - 1) / 2) {
        second = 2 * (second + 1);
        if (heap_comp(h.data[second], h.data[second - 1])) second--;
        h.data[hole] = h.data[second];
        hole         = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
        second       = 2 * (second + 1);
        h.data[hole] = h.data[second - 1];
        hole         = second - 1;
    }
    // __push_heap(first, hole, topIndex = 0, value)
    int64_t parent = (hole - 1) / 2;
    while (hole > 0 && heap_comp(h.data[parent], value)) {
        h.data[hole] = h.data[parent];
        hole         = parent;
        parent       = (hole - 1) / 2;
    }
    h.data[hole] = value;
    return top;
}

// How far from the cells of its batch one update() reaches, in cells on each axis, with R = ceil(l2_max * scale), the reach of the map
// (a valid cell lies less than R from its obstacle, so at most R - 1 on each axis).  On a map that update() left consistent, every cell
// it writes or queues lies within R of a batch cell: the cells of an added obstacle, the cells whose removed obstacle raise() clears,
// and the neighbours of those.  lower() and raise() also read the obstacle of the cells they visit and of their neighbours (one more
// cell out), which lie up to R - 1 further: 2R covers every cell one update() touches.
LAMA_HD uint32_t brushfire_reach(uint32_t radius) { return 2 * radius; }

// Map policy requirements:
//   uint32_t* cell(uint32_t x, uint32_t y)  -- the MUTABLE Map::get (map.cpp:371-412): allocates the
//        patch on first touch, detaches a shared patch, marks the cell known; never returns null
//        (out-of-window accesses return a scratch cell and raise an error bit).
//   DirWindow window
template <typename Map>
struct Brushfire {
    Map& map;
    Heap raise_q, lower_q;
    uint32_t max_sqdist;
    uint32_t err = 0;

    LAMA_HD Brushfire(Map& m, Heap r, Heap l, uint32_t msq) : map(m), raise_q(r), lower_q(l), max_sqdist(msq) {}

    LAMA_HD void push(Heap& q, uint32_t prio, uint32_t x, uint32_t y)
    {
        if (!heap_push(q, heap_entry(prio, cell_key(map.window, x, y)))) err |= kErrHeapOverflow;
    }

    // dynamic_distance_map.cpp:212-226
    LAMA_HD void add_obstacle(uint32_t x, uint32_t y)
    {
        uint32_t* c = map.cell(x, y);
        uint32_t w  = *c;
        if ((w & kDmValid) && dm_sqdist(w) == 0) return;
        *c = dm_pack(0, 0, 0, true, true);
        push(lower_q, 0, x, y);
    }
    // :228-242
    LAMA_HD void remove_obstacle(uint32_t x, uint32_t y)
    {
        uint32_t* c = map.cell(x, y);
        uint32_t w  = *c;
        if (!((w & kDmValid) && dm_sqdist(w) == 0)) return;
        *c = dm_pack(0, 0, 0, false, true);
        push(raise_q, 0, x, y);
    }

    // :244-279 ; neighbour order (+1,0),(0,+1),(-1,0),(0,-1) (:40-43)
    LAMA_HD void raise(uint32_t x, uint32_t y, uint32_t* cur)
    {
        const int dx[4] = {1, 0, -1, 0}, dy[4] = {0, 1, 0, -1};
        for (int i = 0; i < 4; ++i) {
            uint32_t nx = x + dx[i], ny = y + dy[i];
            uint32_t* nb = map.cell(nx, ny);
            uint32_t n   = *nb;
            if ((n & kDmQueued) || !(n & kDmValid)) continue;
            uint32_t* ob = map.cell(nx + dm_ox(n), ny + dm_oy(n));
            if (!(*ob & kDmValid)) {
                push(raise_q, dm_sqdist(n), nx, ny);
                *nb = dm_pack(0, 0, 0, false, true);
            } else {  // `else if (not neighbor->is_queued)` is always taken here
                push(lower_q, dm_sqdist(n), nx, ny);
                *nb = n | kDmQueued;
            }
        }
        *cur &= ~kDmQueued;
    }

    // :281-330
    LAMA_HD void lower(uint32_t x, uint32_t y, uint32_t* cur)
    {
        uint32_t c = *cur;
        if (!(c & kDmQueued)) return;
        const int cox = dm_ox(c), coy = dm_oy(c);
        const int dx[4] = {1, 0, -1, 0}, dy[4] = {0, 1, 0, -1};
        for (int i = 0; i < 4; ++i) {
            if (dx[i] * cox > 0 || dy[i] * coy > 0) continue;  // only update away from the obstacle (:296)
            uint32_t nx = x + dx[i], ny = y + dy[i];
            uint32_t* nb = map.cell(nx, ny);
            uint32_t n   = *nb;
            // obstacle of the current cell, relative to the neighbour
            int rx = cox - dx[i], ry = coy - dy[i];
            uint32_t new_sq = (uint32_t)(rx * rx + ry * ry);
            uint32_t cmp_sq = (n & kDmValid) ? dm_sqdist(n) : max_sqdist;
            bool overwrite  = new_sq < cmp_sq;
            if (!overwrite && new_sq == dm_sqdist(n)) {
                uint32_t o = *map.cell(nx + dm_ox(n), ny + dm_oy(n));
                if (!(n & kDmValid) || !((o & kDmValid) && dm_sqdist(o) == 0)) overwrite = true;
            }
            if (overwrite) {
                push(lower_q, new_sq, nx, ny);
                *nb = dm_pack(new_sq, rx, ry, true, true);
            }
        }
        *cur &= ~kDmQueued;
    }

    // :160-197 ; returns number_of_proccessed_cells
    LAMA_HD uint32_t update()
    {
        uint32_t processed = 0;
        while (raise_q.size) {
            uint32_t key = heap_key(heap_pop(raise_q));
            uint32_t x = key_x(map.window, key), y = key_y(map.window, key);
            uint32_t* cur = map.cell(x, y);
            ++processed;
            raise(x, y, cur);
        }
        while (lower_q.size) {
            uint32_t key = heap_key(heap_pop(lower_q));
            uint32_t x = key_x(map.window, key), y = key_y(map.window, key);
            uint32_t* cur = map.cell(x, y);
            ++processed;
            uint32_t c = *cur;
            if (c & kDmValid) {
                uint32_t o = *map.cell(x + dm_ox(c), y + dm_oy(c));
                if (dm_sqdist(o) == 0) lower(x, y, cur);
            }
        }
        return processed;
    }
};

}  // namespace lama_b200
