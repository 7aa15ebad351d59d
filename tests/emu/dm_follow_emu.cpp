// Test-only host build of dm_follow.h: the chunk windows of a following distance-map update and the extent directory's window.
#include <cstdint>
#include <vector>

#include "../../iris_lama_b200/csrc/dm_follow.h"

using namespace lama_b200;

extern "C" {

uint32_t emu_brushfire_reach(uint32_t radius) { return brushfire_reach(radius); }

// plan_dm_chunks from window {base_px, base_py, dim} over n cells (x, y pairs) in chunks of `chunk`; groups as (first chunk, chunks,
// base x, base y) quadruples in out (room for 4 per chunk), their number in *n_groups; boxes (lo x, lo y, hi x, hi y per chunk) in
// out_boxes.  Returns -1 or the refused chunk's index.
int emu_plan_dm_chunks(int32_t base_px, int32_t base_py, int32_t dim, const uint32_t* cells, int n, int chunk, uint32_t reach, int32_t* out,
                       int* n_groups, int64_t* out_boxes)
{
    std::vector<CellBox> b;
    std::vector<RenderGroup> g;
    const int rc = plan_dm_chunks(DirWindow{base_px, base_py, dim}, cells, n, chunk, reach, b, g);
    for (size_t i = 0; i < g.size(); ++i) {
        out[4 * i] = g[i].first;
        out[4 * i + 1] = g[i].count;
        out[4 * i + 2] = g[i].window.base_px;
        out[4 * i + 3] = g[i].window.base_py;
    }
    for (size_t i = 0; i < b.size(); ++i) {
        out_boxes[4 * i] = b[i].lo[0]; out_boxes[4 * i + 1] = b[i].lo[1]; out_boxes[4 * i + 2] = b[i].hi[0]; out_boxes[4 * i + 3] = b[i].hi[1];
    }
    *n_groups = (int)g.size();
    return rc;
}

int64_t emu_box_patches(const int64_t* box) { return box_patches(CellBox{{box[0], box[1]}, {box[2], box[3]}}); }

// extent_window of cell bounds {mn, mx} with n_patches patches; out = base x, base y, dim
int emu_extent_window(const uint32_t* mn, const uint32_t* mx, int n_patches, int32_t* out)
{
    DirWindow w{-1, -1, -1};
    const int rc = extent_window(mn, mx, n_patches, &w);
    out[0] = w.base_px; out[1] = w.base_py; out[2] = w.dim;
    return rc;
}

int32_t emu_extent_cap() { return kExtentMaxPatches; }

}  // extern "C"
