// render_plan.h -- which scans of a render go through which directory window, and how far the pool of a render-only map grows
// (Engine::render_scans with following on, Engine::grow_pool).  Plain host C++; the CPU tests run it through tests/emu/render_plan_emu.cpp.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

#include "lama_core.h"
#include "ray_core.h"

namespace lama_b200 {

// an inclusive box of cells
struct CellBox {
    int64_t lo[2], hi[2];
};

// The cells one posed scan can touch: its hit cells and its ray start (tf.translation(), as beam_cells computes them), grown by one
// cell of slack.  A ray is a segment, so the box of its two ends holds every cell of its walk, the 3-axis walk of a tilted sensor too.
inline CellBox render_scan_box(const Affine& tf, double scale, const double* pts, int64_t n)
{
    ScanParams sp{};
    sp.scale = scale;
    const double zero[3] = {0.0, 0.0, 0.0};
    const BeamCells s = beam_cells(tf, sp, zero);
    CellBox b{{s.from[0], s.from[1]}, {s.from[0], s.from[1]}};
    for (int64_t i = 0; i < n; ++i) {
        const BeamCells c = beam_cells(tf, sp, pts + 3 * i);
        for (int k = 0; k < 2; ++k) {
            b.lo[k] = std::min<int64_t>(b.lo[k], c.to[k]);
            b.hi[k] = std::max<int64_t>(b.hi[k], c.to[k]);
        }
    }
    for (int k = 0; k < 2; ++k) {
        b.lo[k] -= 1;
        b.hi[k] += 1;
    }
    return b;
}

// every patch the box touches is in window w
inline bool box_in_window(const DirWindow& w, const CellBox& b)
{
    const int64_t base[2] = {w.base_px, w.base_py};
    for (int k = 0; k < 2; ++k)
        if ((b.lo[k] >> kPatchLog2) < base[k] || (b.hi[k] >> kPatchLog2) >= base[k] + w.dim) return false;
    return true;
}

// The patch-aligned dim x dim window centred on the box's patches.  False when no window holds the box: it spans more than dim
// patches on an axis (a box up to dim * 32 cells wide that straddles patch borders can span dim + 1), or it leaves the map's cells.
inline bool render_window_for(const CellBox& b, int32_t dim, DirWindow* out)
{
    const int64_t max_base = ((int64_t)1 << (32 - kPatchLog2)) - dim;
    int64_t base[2];
    for (int k = 0; k < 2; ++k) {
        const int64_t lo = b.lo[k] >> kPatchLog2, hi = b.hi[k] >> kPatchLog2, span = hi - lo + 1;
        if (b.lo[k] < 0 || span > dim) return false;
        base[k] = std::min(std::max<int64_t>(lo - (dim - span) / 2, 0), max_base);
        if (hi >= base[k] + dim) return false;
    }
    *out = DirWindow{(int32_t)base[0], (int32_t)base[1], dim};
    return true;
}

// scans [first, first + count) render through `window`
struct RenderGroup {
    int first, count;
    DirWindow window;
};

// Splits n scans, in order, into groups of consecutive scans that each fit one window: the current window is kept while the next scan's
// box fits it, otherwise the next window is the one render_window_for centres on that scan's box.  Every scan is checked before any
// group is emitted: returns -1 with the groups, or the index of the first scan no window holds, with `groups` empty.  Scans that all fit
// `cur` give one group in `cur`.
inline int plan_render(const DirWindow& cur, const CellBox* boxes, int n, std::vector<RenderGroup>& groups)
{
    groups.clear();
    DirWindow w = cur;
    for (int k = 0; k < n; ++k)
        if (!render_window_for(boxes[k], cur.dim, &w)) return k;
    w = cur;
    for (int k = 0; k < n; ++k) {
        const bool fits = box_in_window(w, boxes[k]);
        if (!fits) render_window_for(boxes[k], cur.dim, &w);
        if (k == 0 || !fits) groups.push_back(RenderGroup{k, 0, w});
        ++groups.back().count;
    }
    return -1;
}

// The largest pool a render-only map grows to: the 24-bit slot field of a directory entry, all ones meaning "not writable".
constexpr int64_t kPoolSlotCap = (int64_t)kDirSlotMask - 1;

// The pool size before a group that may fill all dim2 entries of its window, `held` slots being held outside it (parked): unchanged
// while held + dim2 slots fit or the pool may not grow (an explicit pool size is a hard cap), otherwise doubled until they fit, at most
// kPoolSlotCap.
inline int64_t pool_growth(int64_t n_slots, int64_t held, int64_t dim2, bool growable)
{
    if (!growable || n_slots - held >= dim2 || n_slots >= kPoolSlotCap) return n_slots;
    int64_t n = n_slots < 1 ? 1 : n_slots;
    while (n < held + dim2) n *= 2;
    return std::min(n, kPoolSlotCap);
}

}  // namespace lama_b200
