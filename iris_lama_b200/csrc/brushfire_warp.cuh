// brushfire_warp.cuh -- device implementation of DynamicDistanceMap::update() for one warp per particle.
//
// Semantics are exactly those of ddm_core.h (which the host emulation tests against the oracle): the same pops in
// the same libstdc++ heap order, the same cell writes, the same pushes in the same order.  What changes is the
// schedule inside one pop: the single logical thread of the reference touches its four neighbours one after the
// other; here lanes 0-3 fetch the four neighbour cells (and, where the algorithm asks for it, the neighbours'
// obstacle cells) concurrently and the results are committed in neighbour order 0..3, so that heap pushes happen in
// the reference's order.  A single warp per SM sub-partition is bound by instruction and memory latency, so cutting
// the dependent chain per pop is what matters.
//
// Why the concurrent reads are safe (reference: src/sdm/dynamic_distance_map.cpp:244-330):
//   lower(): neighbour i only ever writes its own cell.  The only foreign cell a later neighbour j reads is the
//     obstacle cell of j, tested for "valid && sqdist == 0".  A cell written by lower() ends with sqdist >= 1 and
//     an obstacle cell (sqdist 0) is never overwritten (new_sqdist >= 1 is neither < 0 nor == 0), so that predicate
//     cannot be changed by an earlier neighbour of the same call.
//   raise(): an earlier neighbour may be cleared (valid = 0); a later neighbour's obstacle test reads `valid`, so
//     the obstacle word is re-read at commit time, after the earlier commits of the same call are visible.
#pragma once

#include "ddm_core.h"
#include "device_store.cuh"

namespace lama_b200 {

constexpr unsigned kFullMask = 0xffffffffu;

// Binary heap with libstdc++ push_heap / pop_heap move order (see ddm_core.h), stored with a one-slot offset so
// that the two children of a node form an aligned 16-byte pair and are fetched with ONE shared-memory load.
// Two levels: the heap starts in shared memory (`slot`); a push that finds either heap of a brushfire full moves both once
// to the particle's regions in global memory (`spill`, same layout) and the brushfire carries on there with the same
// indices (WarpBrushfire::push_spilled).  The two levels run separate instantiations of the brushfire, so that the shared
// one keeps its shared-memory loads and stores.
struct SmemHeap {
    uint64_t* slot;      // shared memory: element j lives in slot[j + 1]; 16-byte aligned
    uint32_t size, cap;  // cap: entries in shared memory (0 once the heap has moved: every shared-level push then fails)
    uint64_t* spill;     // the global region
    uint32_t spill_cap;  // its capacity in entries: the heap's total capacity

    __device__ __forceinline__ static bool push_at(uint64_t* slot, uint32_t& size, uint32_t cap, uint64_t value)
    {
        if (size >= cap) return false;
        int hole = (int)size++;
        while (hole > 0) {
            int parent = (hole - 1) >> 1;
            uint64_t pv = slot[parent + 1];
            if (!heap_comp(pv, value)) break;
            slot[hole + 1] = pv;
            hole = parent;
        }
        slot[hole + 1] = value;
        return true;
    }
    __device__ __forceinline__ static uint64_t pop_at(uint64_t* slot, uint32_t& size)
    {
        const uint64_t t = slot[1];
        const uint32_t last = --size;
        if (last == 0) return t;
        const uint64_t value = slot[last + 1];
        const int len = (int)last;
        int hole = 0, second = 0;
        const int lim = (len - 1) >> 1;
        while (second < lim) {
            second = 2 * (second + 1);
            // children `second - 1` (left) and `second` (right) sit in slots second, second + 1
            const ulonglong2 ch = *reinterpret_cast<const ulonglong2*>(slot + second);
            uint64_t pick = ch.y;
            if (heap_comp(ch.y, ch.x)) {  // comp(right, left): take the left child
                pick = ch.x;
                second--;
            }
            slot[hole + 1] = pick;
            hole = second;
        }
        if ((len & 1) == 0 && second == ((len - 2) >> 1)) {
            second = 2 * (second + 1);
            slot[hole + 1] = slot[second];  // element second - 1
            hole = second - 1;
        }
        while (hole > 0) {
            int parent = (hole - 1) >> 1;
            uint64_t pv = slot[parent + 1];
            if (!heap_comp(pv, value)) break;
            slot[hole + 1] = pv;
            hole = parent;
        }
        slot[hole + 1] = value;
        return t;
    }
    template <bool kGlobal> __device__ __forceinline__ uint64_t pop() { return kGlobal ? pop_at(spill, size) : pop_at(slot, size); }
};

struct WarpBrushfire {
    const StoreView& s;
    int32_t* dir;        // shared-memory copy of the distance-map directory (entries carry kDirOwn)
    int32_t* gdir;
    uint32_t* scratch;   // 32 words: out-of-window / failed accesses land here (one word per lane)
    const uint32_t side;     // window side in cells (dim * 32); all coordinates below are WINDOW-RELATIVE
    const int log2dim;
    const int lane;
    SmemHeap lower_q, raise_q;
    const uint32_t max_sqdist;
    uint32_t err;
    bool dead;           // the pool ran dry: stop touching the map
    bool spilled;        // both heaps live in global memory
#ifdef LAMA_PHASE_TIMING
    long long cyc[6] = {0, 0, 0, 0, 0, 0};   // pop, current + obstacle cell, neighbour fetch, obstacle-of-neighbour check, commit (pushes + stores), pushes alone
#define BF_CLK(v) const long long v = clock64()
#define BF_ACC(k, a, b) cyc[k] += (b) - (a)
#else
#define BF_CLK(v) do { } while (0)
#define BF_ACC(k, a, b) do { } while (0)
#endif

    __device__ WarpBrushfire(const StoreView& sv, int32_t* d, int32_t* g, uint32_t* sc, int l, SmemHeap lo, SmemHeap ra, uint32_t msq)
        : s(sv), dir(d), gdir(g), scratch(sc), side((uint32_t)sv.window.dim * kPatchLen), log2dim(ilog2(sv.window.dim)), lane(l), lower_q(lo),
          raise_q(ra), max_sqdist(msq), err(0), dead(false), spilled(false) {}

    __host__ __device__ static int ilog2(int v)
    {
        int l = 0;
        while ((1 << (l + 1)) <= v) ++l;
        return l;
    }
    // window-relative cell coordinates: key = y << 16 | x (lama_core.h cell_key); unsigned wrap makes x - 1 at the
    // border fall outside `side`
    __device__ __forceinline__ static uint32_t key_of(uint32_t x, uint32_t y) { return (y << 16) | (x & 0xFFFFu); }
    __device__ __forceinline__ int dindex(uint32_t x, uint32_t y) const
    {
        return (x < side && y < side) ? (int)(((y >> kPatchLog2) << log2dim) | (x >> kPatchLog2)) : -1;
    }
    __device__ __forceinline__ uint32_t* cellptr(int entry, uint32_t x, uint32_t y) const
    {
        return s.pool + ((((uint32_t)entry & (uint32_t)kDirSlotMask) << (2 * kPatchLog2)) | cell_index(x, y));
    }

    // ---- mutable Map::get -------------------------------------------------------------------------------------
    __device__ __forceinline__ bool entry_ready(int e) const { return e >= 0 && (e & kDirOwn); }

    // all lanes, identical di: allocate / detach / verify sole ownership (sets kDirOwn in both directory copies)
    __device__ __forceinline__ bool ensure(int di)
    {
        int slot = warp_make_exclusive(s, dir, gdir, di, lane);
        if (slot < 0) {
            err |= kErrPoolEmpty;
            dead = true;
            return false;
        }
        return true;
    }
    // warp-uniform coordinates
    __device__ __forceinline__ uint32_t* uptr(uint32_t x, uint32_t y)
    {
        const int di = dindex(x, y);
        if (di < 0 || dead) {
            if (di < 0) err |= kErrWindow;
            scratch[lane] = 0;
            return &scratch[lane];
        }
        int e = dir[di];
        if (!entry_ready(e)) {
            if (!ensure(di)) {
                scratch[lane] = 0;
                return &scratch[lane];
            }
            e = dir[di];
        }
        return cellptr(e, x, y);
    }
    // per-lane coordinates; inactive lanes get their scratch word
    __device__ __forceinline__ uint32_t* lptr(uint32_t x, uint32_t y, bool active)
    {
        const int di = active ? dindex(x, y) : -1;
        if (active && di < 0) err |= kErrWindow;
        int e = di >= 0 ? dir[di] : -1;
        unsigned m = __ballot_sync(kFullMask, di >= 0 && !entry_ready(e));
        while (m && !dead) {  // rare: first touch of a patch by this particle
            const int l = __ffs(m) - 1;
            ensure(__shfl_sync(kFullMask, di, l));
            e = di >= 0 ? dir[di] : -1;
            m = __ballot_sync(kFullMask, di >= 0 && !entry_ready(e));
        }
        if (!entry_ready(e) || dead) {
            scratch[lane] = 0;
            return &scratch[lane];
        }
        return cellptr(e, x, y);
    }
    // Pointer to cell (x + dx, y + dy) given the pointer `base` to cell (x, y), valid when the target lies in the
    // same patch (which the caller already owns): plain pointer arithmetic, no directory lookup.
    __device__ __forceinline__ static bool same_patch(uint32_t x, uint32_t y, int dx, int dy)
    {
        return (uint32_t)((int)(x & (kPatchLen - 1)) + dx) < (uint32_t)kPatchLen && (uint32_t)((int)(y & (kPatchLen - 1)) + dy) < (uint32_t)kPatchLen;
    }
    // neighbour / obstacle pointer: fast path inside the patch of `base`, directory path otherwise
    __device__ __forceinline__ uint32_t* rel_uptr(uint32_t* base, uint32_t x, uint32_t y, int dx, int dy)
    {
        if (same_patch(x, y, dx, dy) && !is_scratch(base)) return base + dx + dy * kPatchLen;
        return uptr(x + dx, y + dy);
    }
    // per-lane variant; `interior` (warp-uniform) = the whole 4-neighbourhood of (x, y) is inside the patch
    __device__ __forceinline__ uint32_t* rel_lptr(uint32_t* base, bool interior, uint32_t x, uint32_t y, int dx, int dy, bool active)
    {
        if (interior && !is_scratch(base)) return active ? base + dx + dy * kPatchLen : &scratch[lane];
        return lptr(x + dx, y + dy, active);
    }
    __device__ __forceinline__ bool is_scratch(const uint32_t* p) const { return p >= scratch && p < scratch + 32; }
    __device__ __forceinline__ static bool interior_cell(uint32_t x, uint32_t y)
    {
        return ((x & (kPatchLen - 1)) - 1u) < (uint32_t)(kPatchLen - 2) && ((y & (kPatchLen - 1)) - 1u) < (uint32_t)(kPatchLen - 2);
    }

    // read a cell the way the mutable get does: the Container bit ("known") is switched on
    __device__ __forceinline__ uint32_t touch(uint32_t* p)
    {
        uint32_t w = *p;
        if (!(w & kDmKnown)) {
            w |= kDmKnown;
            *p = w;
        }
        return w;
    }

    // A push that found its heap's shared part full (all lanes, warp-uniform): the first one copies both heaps to global memory
    // and sets their shared capacities to 0, so that every later push of the shared-level code lands here too.
    __device__ __forceinline__ void push_spilled(SmemHeap& q, uint64_t value)
    {
        if (!spilled) {
            for (uint32_t j = lane; j < lower_q.size; j += 32) lower_q.spill[j + 1] = lower_q.slot[j + 1];
            for (uint32_t j = lane; j < raise_q.size; j += 32) raise_q.spill[j + 1] = raise_q.slot[j + 1];
            __syncwarp();
            lower_q.cap = raise_q.cap = 0;
            spilled = true;
        }
        if (!SmemHeap::push_at(q.spill, q.size, q.spill_cap, value)) err |= kErrHeapOverflow;
    }
    template <bool kGlobal> __device__ __forceinline__ void push(SmemHeap& q, uint32_t prio, uint32_t key)
    {
        if (kGlobal) {
            if (!SmemHeap::push_at(q.spill, q.size, q.spill_cap, heap_entry(prio, key))) err |= kErrHeapOverflow;
        } else if (!SmemHeap::push_at(q.slot, q.size, q.cap, heap_entry(prio, key))) {
            push_spilled(q, heap_entry(prio, key));
        }
    }

    // dynamic_distance_map.cpp:212-226 / :228-242 (warp-uniform)
    __device__ __forceinline__ void add_obstacle(uint32_t x, uint32_t y)
    {
        uint32_t* c = uptr(x, y);
        const uint32_t w = touch(c);
        if ((w & kDmValid) && dm_sqdist(w) == 0) return;
        *c = dm_pack(0, 0, 0, true, true);
        push<false>(lower_q, 0, key_of(x, y));
    }
    __device__ __forceinline__ void remove_obstacle(uint32_t x, uint32_t y)
    {
        uint32_t* c = uptr(x, y);
        const uint32_t w = touch(c);
        if (!((w & kDmValid) && dm_sqdist(w) == 0)) return;
        *c = dm_pack(0, 0, 0, false, true);
        push<false>(raise_q, 0, key_of(x, y));
    }

    // :244-279
    template <bool G> __device__ __forceinline__ void raise(uint32_t x, uint32_t y, uint32_t* cur)
    {
        const int i = lane & 3;
        const bool act = lane < 4;
        const int dxi = (i == 0) - (i == 2), dyi = (i == 1) - (i == 3);
        const uint32_t nx = x + dxi, ny = y + dyi;
        uint32_t* p = rel_lptr(cur, interior_cell(x, y), x, y, dxi, dyi, act);
        uint32_t n = 0;
        if (act) n = touch(p);
        const bool go = act && !((n & kDmQueued) || !(n & kDmValid));
        uint32_t* po = lptr(nx + dm_ox(n), ny + dm_oy(n), go);
        if (go) touch(po);
        __syncwarp();
        const uint32_t key = key_of(nx, ny);
        for (int j = 0; j < 4; ++j) {
            uint32_t o = 0;
            if (lane == j && go) o = *po;  // re-read: an earlier neighbour of this call may have been cleared
            const bool g   = __shfl_sync(kFullMask, (int)go, j) != 0;
            if (!g) continue;
            const bool clr = __shfl_sync(kFullMask, (int)!(o & kDmValid), j) != 0;
            const uint32_t k  = __shfl_sync(kFullMask, key, j);
            const uint32_t pr = __shfl_sync(kFullMask, dm_sqdist(n), j);
            if (clr) {
                push<G>(raise_q, pr, k);
                if (lane == j) *p = dm_pack(0, 0, 0, false, true);
            } else {  // `else if (not neighbor->is_queued)` is always taken here
                push<G>(lower_q, pr, k);
                if (lane == j) *p = n | kDmQueued;
            }
            __syncwarp();
        }
        if (lane == 0) *cur &= ~kDmQueued;
        __syncwarp();
    }

    // :281-330 ; `c` is the current cell word, known to be queued
    template <bool G> __device__ __forceinline__ void lower(uint32_t x, uint32_t y, uint32_t* cur, uint32_t c)
    {
        const int cox = dm_ox(c), coy = dm_oy(c);
        const int i = lane & 3;
        const int dxi = (i == 0) - (i == 2), dyi = (i == 1) - (i == 3);
        const bool go = lane < 4 && !(dxi * cox > 0 || dyi * coy > 0);  // only update away from the obstacle (:296)
        const uint32_t nx = x + dxi, ny = y + dyi;
        BF_CLK(c0);
        uint32_t* p = rel_lptr(cur, interior_cell(x, y), x, y, dxi, dyi, go);
        uint32_t n = 0;
        if (go) n = touch(p);
#ifdef LAMA_PHASE_TIMING
        n = __shfl_sync(kFullMask, n, lane);   // wait for the load, so that the split below means something
#endif
        BF_CLK(c1);
        BF_ACC(2, c0, c1);
        const int rx = cox - dxi, ry = coy - dyi;
        const uint32_t new_sq = (uint32_t)(rx * rx + ry * ry);
        const uint32_t cmp_sq = (n & kDmValid) ? dm_sqdist(n) : max_sqdist;
        bool over = go && new_sq < cmp_sq;
        const bool chk = go && !over && new_sq == dm_sqdist(n);
        if (__any_sync(kFullMask, chk)) {
            uint32_t* po = lptr(nx + dm_ox(n), ny + dm_oy(n), chk);
            if (chk) {
                const uint32_t o = touch(po);
                if (!(n & kDmValid) || !((o & kDmValid) && dm_sqdist(o) == 0)) over = true;
            }
        }
        __syncwarp();
        unsigned m = __ballot_sync(kFullMask, over) & 0xFu;
        BF_CLK(c2);
        BF_ACC(3, c1, c2);
        const uint32_t key = key_of(nx, ny);
        while (m) {
            const int l = __ffs(m) - 1;
            m &= m - 1;
            BF_CLK(c4);
            push<G>(lower_q, __shfl_sync(kFullMask, new_sq, l), __shfl_sync(kFullMask, key, l));
            BF_CLK(c5);
            BF_ACC(5, c4, c5);
            if (lane == l) *p = dm_pack(new_sq, rx, ry, true, true);
        }
        if (lane == 0) *cur = c & ~kDmQueued;
        __syncwarp();
        BF_CLK(c3);
        BF_ACC(4, c2, c3);
    }

    // :160-197 at one heap level; returns true when the heaps moved to global memory (the caller continues with G = true)
    template <bool G> __device__ __forceinline__ bool run(uint32_t& processed)
    {
        while (raise_q.size) {
            if (!G && spilled) return true;
            const uint32_t key = heap_key(raise_q.pop<G>());
            const uint32_t x = key & 0xFFFFu, y = key >> 16;
            uint32_t* cur = uptr(x, y);
            touch(cur);
            ++processed;
            raise<G>(x, y, cur);
        }
        while (lower_q.size) {
            if (!G && spilled) return true;
            BF_CLK(a0);
            const uint32_t key = heap_key(lower_q.pop<G>());
            BF_CLK(a1);
            BF_ACC(0, a0, a1);
            const uint32_t x = key & 0xFFFFu, y = key >> 16;
            uint32_t* cur = uptr(x, y);
            const uint32_t c = touch(cur);
            ++processed;
            if (c & kDmValid) {
                const uint32_t o = touch(rel_uptr(cur, x, y, dm_ox(c), dm_oy(c)));
                BF_CLK(a2);
                BF_ACC(1, a1, a2);
                if (dm_sqdist(o) == 0 && (c & kDmQueued)) lower<G>(x, y, cur, c);
            }
        }
        return false;
    }
    __device__ __forceinline__ uint32_t update()
    {
        uint32_t processed = 0;
        if (run<false>(processed)) run<true>(processed);
        return processed;
    }
};

}  // namespace lama_b200
