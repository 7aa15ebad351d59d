// Test-only host build of render_plan.h: the grouping of a following render and the pool growth of a render-only map.
#include <cstdint>
#include <vector>

#include "../../iris_lama_b200/csrc/render_plan.h"

using namespace lama_b200;

extern "C" {

// plan_render from window {base_px, base_py, dim} over n boxes (lo x, lo y, hi x, hi y in cells); groups as (first, count, base x, base y)
// quadruples in out (room for 4 n), their number in *n_groups.  Returns -1 or the refused scan's index.
int emu_plan_render(int32_t base_px, int32_t base_py, int32_t dim, const int64_t* boxes, int n, int32_t* out, int* n_groups)
{
    std::vector<CellBox> b((size_t)n);
    for (int k = 0; k < n; ++k) b[k] = CellBox{{boxes[4 * k], boxes[4 * k + 1]}, {boxes[4 * k + 2], boxes[4 * k + 3]}};
    std::vector<RenderGroup> g;
    const int rc = plan_render(DirWindow{base_px, base_py, dim}, b.data(), n, g);
    for (size_t i = 0; i < g.size(); ++i) {
        out[4 * i] = g[i].first;
        out[4 * i + 1] = g[i].count;
        out[4 * i + 2] = g[i].window.base_px;
        out[4 * i + 3] = g[i].window.base_py;
    }
    *n_groups = (int)g.size();
    return rc;
}

int64_t emu_pool_growth(int64_t n_slots, int64_t used, int64_t dim2, int growable) { return pool_growth(n_slots, used, dim2, growable != 0); }

// render_scan_box of n points (xyz) seen from pose (x, y, theta) through an identity sensor transform; out = lo x, lo y, hi x, hi y
void emu_render_scan_box(const double* xyr, const double* pts, int n, double scale, int64_t* out)
{
    MovingTf m{};
    m.l[0] = m.l[4] = m.l[8] = 1.0;
    const CellBox b = render_scan_box(compose_tf(se2_from_xyr(xyr[0], xyr[1], xyr[2]), m), scale, pts, n);
    out[0] = b.lo[0]; out[1] = b.lo[1]; out[2] = b.hi[0]; out[3] = b.hi[1];
}

}  // extern "C"
