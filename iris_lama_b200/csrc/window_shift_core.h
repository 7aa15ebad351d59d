// window_shift_core.h -- parked directory entries of the 2-D maps and the per-entry logic of a window shift.  Plain C++ usable
// from host and device: k_shift_count / k_shift_apply (kernels.cu), the lookups of the host-facing read kernels and the test-only
// host emulation (tests/emu/window_shift_emu.cpp) all run these functions.
//
// A map's directory covers a dir_dim x dir_dim window of patches.  When the window moves (Engine::shift_window), the entries it leaves
// are PARKED: kept, with their slot and flag bits unchanged, in a list per (set, particle, kind) sorted by absolute patch coordinate
// (y, then x).  A parked entry holds the reference its directory entry held.  When the window comes back over a parked patch, the
// entry returns to the directory as it was.
#pragma once

#include "lama_core.h"

namespace lama_b200 {

struct ParkEntry {
    int32_t px, py;   // absolute patch coordinates (cell >> 5)
    int32_t entry;    // the directory entry: slot | kDirHot | kDirOwn
};

// (ay, ax) < (by, bx): the order of a parked list
LAMA_HD bool park_before(int32_t ax, int32_t ay, int32_t bx, int32_t by) { return ay < by || (ay == by && ax < bx); }

// first position of a sorted list whose key is not before (px, py)
LAMA_HD int park_lower_bound(const ParkEntry* l, int n, int32_t px, int32_t py)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (park_before(l[m].px, l[m].py, px, py)) lo = m + 1;
        else hi = m;
    }
    return lo;
}

// the parked entry of patch (px, py), or -1
LAMA_HD int32_t park_find(const ParkEntry* l, int n, int32_t px, int32_t py)
{
    const int i = park_lower_bound(l, n, px, py);
    return (i < n && l[i].px == px && l[i].py == py) ? l[i].entry : -1;
}

LAMA_HD bool patch_in_window(const DirWindow& w, int32_t px, int32_t py)
{
    return (unsigned)(px - w.base_px) < (unsigned)w.dim && (unsigned)(py - w.base_py) < (unsigned)w.dim;
}

// directory entry `entry` at index i of window w is parked by a shift to window nw
LAMA_HD bool shift_leaves(const DirWindow& w, const DirWindow& nw, int i, int32_t entry)
{
    return entry >= 0 && !patch_in_window(nw, w.base_px + i % w.dim, w.base_py + i / w.dim);
}

// a parked entry returns to the directory of window nw
LAMA_HD bool shift_enters(const DirWindow& nw, const ParkEntry& a) { return patch_in_window(nw, a.px, a.py); }

// The new directory entry at index j of window nw: from the old directory when the patch was inside the old window w, otherwise
// from the parked list (-1 when the patch is in neither).
LAMA_HD int32_t shift_new_entry(const DirWindow& w, const DirWindow& nw, int j, const int32_t* old_dir, const ParkEntry* parked, int n_parked)
{
    const int32_t px = nw.base_px + j % nw.dim, py = nw.base_py + j / nw.dim;
    if (patch_in_window(w, px, py)) return old_dir[(py - w.base_py) * w.dim + (px - w.base_px)];
    return park_find(parked, n_parked, px, py);
}

// number of patches of window w whose key precedes the key of (px, py), a patch outside w: the rank of a parked entry among the
// directory indices of w, which run in (y, x) order
LAMA_HD int window_rank(const DirWindow& w, int32_t px, int32_t py)
{
    const int r = py - w.base_py;
    if (r < 0) return 0;
    if (r >= w.dim) return w.dim * w.dim;
    return r * w.dim + (px < w.base_px ? 0 : w.dim);
}

// The new parked list is the merge of the old list without the entries that enter (A) and the entries that leave (B, in directory
// order).  leave_before[i] = leaving entries among directory indices < i (dim^2 + 1 values), enter_before[i] = entering entries among
// A[0 .. i) (n_parked + 1 values).
// position of A[i] (which stays parked) in the new list
LAMA_HD int shift_pos_parked(const DirWindow& w, const ParkEntry* parked, int i, const int32_t* enter_before, const int32_t* leave_before)
{
    return (i - enter_before[i]) + leave_before[window_rank(w, parked[i].px, parked[i].py)];
}
// position of the leaving directory entry at index i of window w in the new list
LAMA_HD int shift_pos_leaving(const DirWindow& w, int i, const ParkEntry* parked, int n_parked, const int32_t* enter_before, const int32_t* leave_before)
{
    const int lb = park_lower_bound(parked, n_parked, w.base_px + i % w.dim, w.base_py + i / w.dim);
    return leave_before[i] + (lb - enter_before[lb]);
}

// k_shift_apply writes the enter prefixes of list i (length + 1 values) at scratch offset list offset + i.  A prune shortens lists in
// place, so the arena may have gaps: the scratch needs the end of the furthest list plus one value per list.  ol = {offset, length}
// pairs of n_lists lists.
LAMA_HD int shift_enter_base(int32_t offset, int list) { return offset + list; }
inline size_t shift_scratch_ints(const int32_t* ol, int n_lists)
{
    size_t end = 0;
    for (int i = 0; i < n_lists; ++i) end = end > (size_t)ol[2 * i] + (size_t)ol[2 * i + 1] ? end : (size_t)ol[2 * i] + (size_t)ol[2 * i + 1];
    return end + (size_t)n_lists;
}

}  // namespace lama_b200
