// mc_table.h -- the marching-cubes triangle table of the truncated signed distance map's toMesh, generated on the host from a
// stated rule rather than copied from a published table.  Host-only plain C++.
//
// Cube corners and edges are the reference's (corner order of toMesh's `delta`, MarchingCubes::edge_index_pairs); corner i is
// "negative" (configuration bit i) when sdf[i] < 0.  For configuration c:
//   1. Faces.  On each of the 6 faces, an edge whose two corners differ in sign is a crossing edge.  A face has 0, 2 or 4 of them.
//      Two crossing edges are joined by one segment.  Four (the ambiguous face: negative corners on a diagonal) are joined as two
//      segments, each cutting off one negative corner, so the negative corners are separated.  The rule reads only the face's
//      4 corners, so the two cubes sharing a face make the same segments and the surface has no cracks.
//   2. Direction.  Each segment is directed so that, seen from outside the cube, the negative corners are on its left.  Every
//      crossing edge then ends exactly one segment and starts exactly one other, and the segments chain into closed loops.
//   3. Triangles.  Loops are taken in the order of their lowest edge index; each loop is fan-triangulated from that edge, keeping
//      the loop's direction.  The right-hand normal of every triangle (a, b, c) then points to the negative side, so the reversed
//      faces of the PLY export (export.cpp:138-140) point toward sdf > 0, the side the sensor saw.
// The vertices on crossing edges do not depend on the table; only the choice of triangles does.
#pragma once

#include <cstdint>
#include <stdexcept>

namespace lama_b200 {

constexpr int kMcRow = 16;   // at most 5 triangles + the -1 terminator (checked when the table is built)

struct McTable {
    int8_t tri[256][kMcRow];   // edge indices, 3 per triangle, -1 terminated
    uint8_t ntri[256];
};

inline McTable mc_build_table()
{
    static const int corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
    static const int edge[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6}, {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
    // corners of each face in cyclic order, and its outward normal
    static const int face[6][4] = {{0, 1, 2, 3}, {4, 5, 6, 7}, {0, 1, 5, 4}, {3, 2, 6, 7}, {0, 3, 7, 4}, {1, 2, 6, 5}};
    static const int normal[6][3] = {{0, 0, -1}, {0, 0, 1}, {0, -1, 0}, {0, 1, 0}, {-1, 0, 0}, {1, 0, 0}};
    auto edge_of = [&](int a, int b) {
        for (int e = 0; e < 12; ++e)
            if ((edge[e][0] == a && edge[e][1] == b) || (edge[e][0] == b && edge[e][1] == a)) return e;
        throw std::logic_error("mc table: not an edge");
    };
    McTable t;
    for (int c = 0; c < 256; ++c) {
        auto neg = [c](int i) { return ((c >> i) & 1) != 0; };
        int next[12];
        for (int e = 0; e < 12; ++e) next[e] = -1;
        // a directed segment ea -> eb, oriented so the negative end of ea lies on its left seen from outside face f
        auto add_segment = [&](int f, int ea, int eb) {
            const int p = neg(edge[ea][0]) ? edge[ea][0] : edge[ea][1];
            int ma[3], mb[3], u[3], v[3];
            for (int k = 0; k < 3; ++k) {
                ma[k] = corner[edge[ea][0]][k] + corner[edge[ea][1]][k];   // twice the edge midpoints
                mb[k] = corner[edge[eb][0]][k] + corner[edge[eb][1]][k];
                u[k] = mb[k] - ma[k];
                v[k] = 2 * corner[p][k] - ma[k];
            }
            const int x[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
            const int s = x[0] * normal[f][0] + x[1] * normal[f][1] + x[2] * normal[f][2];
            const int from = s > 0 ? ea : eb, to = s > 0 ? eb : ea;
            if (s == 0 || next[from] != -1) throw std::logic_error("mc table: inconsistent face segments");
            next[from] = to;
        };
        for (int f = 0; f < 6; ++f) {
            int fe[4], nc = 0;
            for (int j = 0; j < 4; ++j) {
                fe[j] = edge_of(face[f][j], face[f][(j + 1) % 4]);
                nc += neg(face[f][j]) != neg(face[f][(j + 1) % 4]);
            }
            if (nc == 2) {
                int ends[2], k = 0;
                for (int j = 0; j < 4; ++j)
                    if (neg(face[f][j]) != neg(face[f][(j + 1) % 4])) ends[k++] = fe[j];
                add_segment(f, ends[0], ends[1]);
            } else if (nc == 4) {
                for (int j = 0; j < 4; ++j)   // cut off each negative corner: its two face edges fe[j - 1] and fe[j]
                    if (neg(face[f][j])) add_segment(f, fe[(j + 3) % 4], fe[j]);
            }
        }
        bool seen[12] = {};
        int n = 0;
        for (int e0 = 0; e0 < 12; ++e0) {
            if (next[e0] < 0 || seen[e0]) continue;
            int loop[12], len = 0;
            for (int e = e0; !seen[e]; e = next[e]) {
                if (next[e] < 0) throw std::logic_error("mc table: open loop");
                seen[e] = true;
                loop[len++] = e;
            }
            for (int i = 1; i + 1 < len; ++i) {
                if (3 * n + 3 >= kMcRow) throw std::logic_error("mc table: row too short");
                t.tri[c][3 * n] = (int8_t)loop[0];
                t.tri[c][3 * n + 1] = (int8_t)loop[i];
                t.tri[c][3 * n + 2] = (int8_t)loop[i + 1];
                ++n;
            }
        }
        for (int k = 3 * n; k < kMcRow; ++k) t.tri[c][k] = -1;
        t.ntri[c] = (uint8_t)n;
    }
    return t;
}

}  // namespace lama_b200
