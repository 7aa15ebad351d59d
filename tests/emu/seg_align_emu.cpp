// seg_align_emu.cpp -- TEST-ONLY host build of the sector-aligned segment partition k_raycast uses for the beams of x-major beam groups
// (ray_core.h xmajor_seg_shift, SegWalk, StrideWalk) against the reference's iterative walk.  Never linked into the product.
#include <cstdint>
#include <random>
#include <vector>

#include "../../iris_lama_b200/csrc/ray_core.h"

using namespace lama_b200;

extern "C" {

// The partition of raycast_pass for a beam of an x-major group (kSegSteps = 64, kXStride = 8), delta = xmajor_seg_shift for an x-major
// beam and 0 for a y-major one: segment 0 walks steps 1 .. 64 - delta one at a time, segment s >= 1 covers s 64 + 1 - delta ..
// (s + 1) 64 - delta with 8 lanes at consecutive offsets and stride 8, and the beam has ceil((n - 1 + delta) / 64) segments.  Checks:
// every step 1 .. n - 1 is visited exactly once and on the reference's cell; in segments >= 1 of an x-major beam, the cells of one
// instruction (the 8 lanes at the same iteration) lie in one aligned octet of x, and the first cell of each such segment starts one
// in walk direction; the look-ahead of the kernel's loop stays inside the bounding box of the beam's end cells.
// Beams: from (c, c) to every cell of a (2 r + 1)^2 square around it when r > 0, else `count` random beams inside a window of `side`
// cells.  Returns the number of beams that fail.
int emu_seg_align_check(int r, uint32_t c, uint32_t seed, int count, int side)
{
    constexpr int kSeg = 64, kStride = 8;
    int bad = 0;
    std::vector<uint32_t> ref_cells;
    std::vector<int> seen;
    auto one = [&](uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty) {
        BeamCells bc;
        bc.from[0] = fx; bc.from[1] = fy; bc.from[2] = 7u;
        bc.to[0] = tx; bc.to[1] = ty; bc.to[2] = 7u;
        bc.mark_hit = true;
        RayWalk ref(bc);
        const int n = ref.n, walk = n - 1;
        ref_cells.assign(1, 0u);   // ref_cells[i] = packed cell of step i (1 .. n - 1)
        while (ref.next()) ref_cells.push_back(ref.x | (ref.y << 16));
        seen.assign(n > 1 ? n : 1, 0);
        const uint32_t x0 = fx < tx ? fx : tx, x1 = fx < tx ? tx : fx, y0 = fy < ty ? fy : ty, y1 = fy < ty ? ty : fy;
        auto in_box = [&](uint32_t P) { return (P & 0xFFFFu) >= x0 && (P & 0xFFFFu) <= x1 && (P >> 16) >= y0 && (P >> 16) <= y1; };
        const uint32_t adx = tx > fx ? tx - fx : fx - tx, ady = ty > fy ? ty - fy : fy - ty;
        const bool xmajor = adx >= ady;
        const int delta = xmajor ? xmajor_seg_shift(fx, tx) : 0;
        const int segs = walk > 0 ? (walk + delta + kSeg - 1) / kSeg : 0;
        bool ok = delta >= 0 && delta < kStride;
        auto visit = [&](int pos, uint32_t P) {
            ok = ok && pos >= 1 && pos <= walk && P == ref_cells[pos];
            if (pos >= 1 && pos <= walk) ++seen[pos];
        };
        if (segs > 0) {
            SegWalk w;
            w.init(fx, fy, tx, ty, 0, kSeg - delta);
            while (w.next()) visit(w.i, w.P);
        }
        for (int s = 1; s < segs; ++s) {
            const int first = s * kSeg + 1 - delta;
            ok = ok && first <= walk;   // no empty segment
            StrideWalk lane[kStride];
            bool live[kStride];
            for (int k = 0; k < kStride; ++k) {
                lane[k].init(fx, fy, tx, ty, first + k, first + kSeg - 1, kStride);
                live[k] = lane[k].i <= lane[k].iend;
            }
            if (xmajor) ok = ok && (lane[0].P & 7u) == (tx < fx ? 7u : 0u);
            for (bool any = true; any;) {
                any = false;
                int octet = -1;
                for (int k = 0; k < kStride; ++k) {
                    if (!live[k]) continue;
                    any = true;
                    visit(lane[k].i, lane[k].P);
                    const int o = (int)((lane[k].P & 0xFFFFu) >> 3);
                    if (xmajor) ok = ok && (octet < 0 || o == octet);
                    octet = o;
                    if (lane[k].i > lane[k].iend - kStride) { live[k] = false; continue; }
                    lane[k].step();
                    ok = ok && in_box(lane[k].P);
                }
            }
        }
        for (int i = 1; i <= walk; ++i) ok = ok && seen[i] == 1;
        if (!ok) ++bad;
    };
    if (r > 0) {
        for (int ty = -r; ty <= r; ++ty)
            for (int tx = -r; tx <= r; ++tx) one(c, c, (uint32_t)((int)c + tx), (uint32_t)((int)c + ty));
    } else {
        std::mt19937 g(seed);
        for (int k = 0; k < count; ++k) one(g() % side, g() % side, g() % side, g() % side);
    }
    return bad;
}

}  // extern "C"
