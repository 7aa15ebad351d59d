// dm_follow.h -- the window decisions of a following 2-D distance map (lama_dm_set_follow, Loc2D): which window each chunk of an
// obstacle update runs in (Engine::dm_apply), and the dense directory over the whole map that global localisation reads
// (Engine::match_extent).  Plain host C++; the CPU tests run it through tests/emu/dm_follow_emu.cpp.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

#include "ddm_core.h"
#include "render_plan.h"

namespace lama_b200 {

// The cells one brushfire of the n cells (x, y pairs) can touch: their box grown by `reach` cells (brushfire_reach).  n >= 1.
inline CellBox dm_chunk_box(const uint32_t* cells_xy, int n, uint32_t reach)
{
    CellBox b{{cells_xy[0], cells_xy[1]}, {cells_xy[0], cells_xy[1]}};
    for (int i = 1; i < n; ++i)
        for (int k = 0; k < 2; ++k) {
            b.lo[k] = std::min<int64_t>(b.lo[k], cells_xy[2 * i + k]);
            b.hi[k] = std::max<int64_t>(b.hi[k], cells_xy[2 * i + k]);
        }
    for (int k = 0; k < 2; ++k) {
        b.lo[k] -= reach;
        b.hi[k] += reach;
    }
    return b;
}

// patches the box touches: the most a brushfire inside it can allocate
inline int64_t box_patches(const CellBox& b)
{
    return ((b.hi[0] >> kPatchLog2) - (b.lo[0] >> kPatchLog2) + 1) * ((b.hi[1] >> kPatchLog2) - (b.lo[1] >> kPatchLog2) + 1);
}

// The windows of an obstacle list of n cells applied in chunks of `chunk` cells (one brushfire each), in list order: groups of
// consecutive chunks that each fit one window, as plan_render splits scans (the current window while it holds the next chunk's box,
// otherwise the window centred on that box).  Every chunk is checked first: returns -1, or the first chunk no window holds with
// `groups` empty.  RenderGroup::first / count count chunks.  `boxes` receives every chunk's box.
inline int plan_dm_chunks(const DirWindow& cur, const uint32_t* cells_xy, int n, int chunk, uint32_t reach, std::vector<CellBox>& boxes,
                          std::vector<RenderGroup>& groups)
{
    boxes.clear();
    for (int done = 0; done < n; done += chunk) boxes.push_back(dm_chunk_box(cells_xy + 2 * (size_t)done, std::min(chunk, n - done), reach));
    return plan_render(cur, boxes.data(), (int)boxes.size(), groups);
}

// The dense directory global localisation reads: a square window over every allocated patch of the map, at most kExtentMaxPatches on
// a side (4096^2 entries of 4 bytes = 64 MiB).
constexpr int32_t kExtentMaxPatches = 4096;

// The extent window of a map whose n_patches allocated patches have the cell bounds {mn, mx} (Engine::bounds: patch aligned, mx
// exclusive): base = the lowest patch on each axis, dim = the larger span.  0: no patch (nothing to build); -1: a span exceeds the cap.
inline int extent_window(const uint32_t mn[2], const uint32_t mx[2], int n_patches, DirWindow* out)
{
    if (n_patches <= 0) return 0;
    int64_t span = 0;
    for (int k = 0; k < 2; ++k) span = std::max<int64_t>(span, (int64_t)(mx[k] >> kPatchLog2) - (int64_t)(mn[k] >> kPatchLog2));
    if (span > kExtentMaxPatches) return -1;
    *out = DirWindow{(int32_t)(mn[0] >> kPatchLog2), (int32_t)(mn[1] >> kPatchLog2), (int32_t)span};
    return 1;
}

}  // namespace lama_b200
