// stride_walk_emu.cpp -- TEST-ONLY host build of ray_core.h's StrideWalk (the walk k_raycast uses for the segments of x-major
// beam groups after the first) against the reference's iterative walk.  Never linked into the product.
#include <cstdint>
#include <random>
#include <vector>

#include "../../iris_lama_b200/csrc/ray_core.h"

using namespace lama_b200;

extern "C" {

// For every segment of `seg` steps and every start offset 0 .. stride - 1, the walk must visit exactly the cells of RayWalk
// (Map::computeRay) at the steps of the segment congruent to the offset, and the kernel's loop (one step ahead while a next cell
// exists) must stay inside the bounding box of the beam's end cells.  Beams: from the centre to every cell of a (2 r + 1)^2 square
// when r > 0, else `count` random beams inside a window of `side` cells.  Returns the number of beams that differ.
int emu_stridewalk_check(int r, uint32_t seed, int count, int side, int seg, int stride)
{
    int bad = 0;
    std::vector<uint32_t> ref_cells;
    auto one = [&](uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty) {
        BeamCells bc;
        bc.from[0] = fx; bc.from[1] = fy; bc.from[2] = 7u;
        bc.to[0] = tx; bc.to[1] = ty; bc.to[2] = 7u;
        bc.mark_hit = true;
        RayWalk ref(bc);
        const int n = ref.n;
        ref_cells.assign(1, 0u);   // ref_cells[i] = packed cell of step i (1 .. n - 1)
        while (ref.next()) ref_cells.push_back(ref.x | (ref.y << 16));
        const uint32_t x0 = fx < tx ? fx : tx, x1 = fx < tx ? tx : fx, y0 = fy < ty ? fy : ty, y1 = fy < ty ? ty : fy;
        auto in_box = [&](uint32_t P) { return (P & 0xFFFFu) >= x0 && (P & 0xFFFFu) <= x1 && (P >> 16) >= y0 && (P >> 16) <= y1; };
        bool ok = true;
        for (int s0 = 0; s0 == 0 || s0 < n - 1; s0 += seg)
            for (int p = 0; p < stride; ++p) {
                StrideWalk w;
                w.init(fx, fy, tx, ty, s0 + 1 + p, s0 + seg, stride);
                int expect = s0 + 1 + p;   // the next step this lane must visit
                if (w.i <= w.iend) {
                    uint32_t P = w.P;
                    const int last_prefetch = w.iend - stride;
                    for (;;) {
                        const int pos = w.i;
                        ok = ok && pos == expect && pos < (int)ref_cells.size() && P == ref_cells[pos];
                        expect += stride;
                        if (pos > last_prefetch) break;
                        w.step();
                        P = w.P;
                        ok = ok && in_box(P);
                    }
                }
                // every step of the segment congruent to the offset was visited, and no other
                const int seg_end = s0 + seg < n - 1 ? s0 + seg : n - 1;
                ok = ok && expect > seg_end && (expect == s0 + 1 + p || expect - stride <= seg_end);
            }
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

}  // extern "C"
