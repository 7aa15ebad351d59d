// ray_core.h -- per-beam geometry, the integer Bresenham walk and the per-cell ordered replay that
// turns parallel counter updates back into the reference's sequential obstacle events.
//
// Reference: PFSlam2D::updateParticleMaps src/pf_slam2d.cpp:439-509 (twin Slam2D::updateMaps
// src/slam2d.cpp:247-321), Map::computeRay src/sdm/map.cpp:198-227,
// FrequencyOccupancyMap::setFree/setOccupied src/sdm/frequency_occupancy_map.cpp:65-91.
//
// How the parallel kernel stays exact.  The reference walks beams 0..N-1 sequentially; for beam i it
// first marks the hit cell (setOccupied) and then every interior ray cell (setFree).  Counter updates
// commute, so all beams add into the packed {occupied, visited} words with atomics.  What does NOT
// commute is (a) at which touch a cell crosses the 0.25 threshold, which decides the
// addObstacle/removeObstacle calls, and (b) the order of those calls, which is the push order of the
// brushfire heaps.  Both only concern cells that receive a hit in this scan or are currently
// distance-map obstacles ("candidate" cells, found with per-patch bitmaps in shared memory); every touch of
// such a cell is logged as (cell, beam, pos, kind), the log
// is sorted, and each cell's touches are replayed in beam order from its pre-scan counters.  The
// obstacle events carry the sequence stamp (beam, pos) of the touch that caused them and are sorted
// by it, which reproduces the reference's call order exactly.
#pragma once

#include "lama_core.h"

namespace lama_b200 {

struct ScanParams {
    MovingTf moving;         // sensor pose in the base frame
    double scale;            // 1 / resolution
    double truncated_ray;    // Options::truncated_ray   (pf_slam2d.h:155)
    double truncated_range;  // Options::truncated_range (pf_slam2d.h:158)
    int n_beams;
    int lo_ray;              // 1: LidarOdometry2D's rule instead of the two above: rays longer than 1 m keep their last metre
                             //    (`if (ray_length >= 1.0) start = hit - AB / ray_length`, lidar_odometry_2d.cpp:103-110)
};

struct BeamCells {
    uint32_t from[3];
    uint32_t to[3];
    bool mark_hit;
};

// pf_slam2d.cpp:463-491 : world hit / ray start of one beam; returns mark_hit.
LAMA_HD bool beam_world(const Affine& tf, const ScanParams& sp, const double* pt, double hit[3], double start[3])
{
    start[0] = tf.t[0]; start[1] = tf.t[1]; start[2] = tf.t[2];
    double AB[3] = {0, 0, 0};
    apply_tf(tf, pt[0], pt[1], pt[2], hit);
    double ray_length = 1.0;
    bool mark_hit = true;
    if (sp.lo_ray) {
        for (int k = 0; k < 3; ++k) AB[k] = add_rn(hit[k], -start[k]);
        ray_length = sqrt(add_rn(add_rn(mul_rn(AB[0], AB[0]), mul_rn(AB[1], AB[1])), mul_rn(AB[2], AB[2])));
        if (ray_length >= 1.0)
            for (int k = 0; k < 3; ++k) start[k] = add_rn(hit[k], -(AB[k] / ray_length));
        return true;
    }
    if (sp.truncated_range > 0.0) {
        for (int k = 0; k < 3; ++k) AB[k] = add_rn(hit[k], -start[k]);
        ray_length = sqrt(add_rn(add_rn(mul_rn(AB[0], AB[0]), mul_rn(AB[1], AB[1])), mul_rn(AB[2], AB[2])));
        if (sp.truncated_range < ray_length) {
            for (int k = 0; k < 3; ++k) hit[k] = add_rn(start[k], mul_rn(AB[k] / ray_length, sp.truncated_range));
            mark_hit = false;
        }
    }
    if (mark_hit && sp.truncated_ray > 0.0) {
        if (sp.truncated_range == 0.0) {
            for (int k = 0; k < 3; ++k) AB[k] = add_rn(hit[k], -start[k]);
            ray_length = sqrt(add_rn(add_rn(mul_rn(AB[0], AB[0]), mul_rn(AB[1], AB[1])), mul_rn(AB[2], AB[2])));
        }
        if (sp.truncated_ray < ray_length)
            for (int k = 0; k < 3; ++k) start[k] = add_rn(hit[k], -mul_rn(AB[k] / ray_length, sp.truncated_ray));
    }
    return mark_hit;
}

// pf_slam2d.cpp:463-499 : the map cells of one beam's ray start and hit.
LAMA_HD BeamCells beam_cells(const Affine& tf, const ScanParams& sp, const double* pt)
{
    double start[3], hit[3];
    BeamCells b;
    b.mark_hit = beam_world(tf, sp, pt, hit, start);
    for (int k = 0; k < 3; ++k) {
        b.to[k]   = w2m(hit[k], sp.scale);
        b.from[k] = w2m(start[k], sp.scale);
    }
    return b;
}

// Map::computeRay (map.cpp:198-227): integer 3-D Bresenham that emits n-1 cells, excluding both
// endpoints.  Usage:  RayWalk w(b); while (w.next()) touch(w.x, w.y);
struct RayWalk {
    int64_t err[3], coord[3], delta[3], step[3];
    int n, i;
    uint32_t x, y;
    LAMA_HD explicit RayWalk(const BeamCells& b)
    {
        n = 0;
        i = 0;
        x = y = 0;
        if (b.from[0] == b.to[0] && b.from[1] == b.to[1] && b.from[2] == b.to[2]) return;
        for (int j = 0; j < 3; ++j) {
            err[j]   = 0;
            coord[j] = (int64_t)b.from[j];
            delta[j] = (int64_t)b.to[j] - coord[j];
            step[j]  = delta[j] < 0 ? -1 : 1;
            delta[j] = delta[j] < 0 ? -delta[j] : delta[j];
        }
        int64_t m = delta[0] > delta[1] ? delta[0] : delta[1];
        n = (int)(m > delta[2] ? m : delta[2]);
    }
    LAMA_HD int cells() const { return n > 0 ? n - 1 : 0; }
    LAMA_HD bool next()
    {
        if (i >= n - 1) return false;
        ++i;
        for (int j = 0; j < 3; ++j) err[j] += delta[j];
        for (int j = 0; j < 3; ++j) {
            if ((err[j] << 1) < n) continue;
            coord[j] += step[j];
            err[j] -= n;
        }
        x = (uint32_t)coord[0];
        y = (uint32_t)coord[1];
        return true;
    }
};

// ---- packed cells: P = yr << 16 | xr, window-relative coordinates (each < 2^13) -------------------------------------------
// directory index of the patch of P in a window of (1 << log2dim)^2 patches
LAMA_HD uint32_t packed_dir_index(uint32_t P, int log2dim) { return ((P >> 21) << log2dim) | ((P >> kPatchLog2) & 0xFFu); }
// byte offset of the cell inside its 4 KiB patch: (x & 31) * 4 + (y & 31) * 128  ==  4 * cell_index(x, y)
LAMA_HD uint32_t packed_cell_offset(uint32_t P) { return ((P << 2) & 0x7Cu) | ((P >> 9) & 0xF80u); }

// ---- the planar walk of the ray-cast kernel ---------------------------------------------------------------------------
// Map::computeRay (map.cpp:198-227) for a planar beam (from.z == to.z: the z axis never moves), started at any step.  The major axis (delta == n) moves on every step: its
// error term returns to 0 each time (err += n; 2 err >= n; err -= n), so only the minor axis carries state:
//   e += d;  if (2 e >= n) { minor coordinate moves; e -= n; }          [kept as e2 = 2 e - n: a sign test]
// (dx == dy: both axes move on every step, which the same update yields with d == n.)
// The cell is kept PACKED, P = yr << 16 | xr (window-relative coordinates, each < 2^13): a step is one addition of a packed
// step vector (sy * 65536 + sx as a signed number; no borrow crosses the halves because all cells of a beam lie inside the
// bounding box of its end cells, which is inside the window), and P is also the key of the ordered-path log.
struct SegWalk {
    // the minor-axis state is kept as e2 = 2 e - n, so that the reference's test 2 e >= n is a sign test: e2 += 2 d; if (e2 >= 0) { move; e2 -= 2 n; }
    int e2, d2, n2, i, iend;
    int M, N;            // packed major / minor step vectors
    uint32_t P;
    LAMA_HD void init(uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty, int i0, int steps)
    {
        const int ddx = (int)(tx - fx), ddy = (int)(ty - fy);
        const int sx = ddx < 0 ? -1 : 1, sy = ddy < 0 ? -1 : 1;
        const int dx = ddx < 0 ? -ddx : ddx, dy = ddy < 0 ? -ddy : ddy;
        const bool xmajor = dx >= dy;
        const int n = xmajor ? dx : dy, d = xmajor ? dy : dx;
        M = xmajor ? sx : sy * 65536;
        N = xmajor ? sy * 65536 : sx;
        d2   = 2 * d;
        n2   = 2 * n;
        i    = i0;
        iend = i0 + steps < n - 1 ? i0 + steps : n - 1;
        uint32_t k = 0;
        int e = 0;
        if (i0 != 0 && n != 0) {  // closed form of the state after i0 steps
            k = (2u * (uint32_t)i0 * (uint32_t)d + (uint32_t)n) / (2u * (uint32_t)n);
            e = i0 * d - (int)k * n;
        }
        e2 = 2 * e - n;
        P  = (fx | (fy << 16)) + (uint32_t)(M * i0 + N * (int)k);
    }
    LAMA_HD void step()   // one step without the end test: callers that count the steps themselves (iend - i of them)
    {
        ++i;
        e2 += d2;
        P += (uint32_t)M;
        if (e2 >= 0) { P += (uint32_t)N; e2 -= n2; }
    }
    LAMA_HD bool next()
    {
        if (i >= iend) return false;
        step();
        return true;
    }
};

// The planar walk taken S steps at a time: it visits the cells SegWalk visits at steps first, first + S, first + 2 S, ... up to
// iend.  With S d = q n + r (0 <= r < n), a stride moves the major axis S times and the minor axis q or q + 1 times: the
// state after step j has e in [-n/2, n/2), so e + r < 3n/2 and one test decides the extra move, as in the unit step
//   e += r;  minor coordinate += q;  if (2 e >= n) { minor coordinate moves once more; e -= n; }
// and a stride costs what a step costs.  k_raycast lets S lanes walk one x-major beam at consecutive offsets: the cells of one
// reduction instruction then lie along a row of each beam's patch instead of down a column.
struct StrideWalk {
    int e2, r2, n2, i, iend, S;   // e2 = 2 e - n as in SegWalk, r2 = 2 r
    int MS, N;                    // packed vector of one stride without the extra minor move / of the extra minor move
    uint32_t P;
    // first >= 1; the walk ends at step min(end, n - 1), the last interior cell; i > iend: nothing to visit
    LAMA_HD void init(uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty, int first, int end, int stride)
    {
        SegWalk w;
        w.init(fx, fy, tx, ty, first, end - first);
        const int n = w.n2 >> 1, d = w.d2 >> 1;
        const int q = n ? (int)((uint32_t)(stride * d) / (uint32_t)n) : 0;
        e2 = w.e2; r2 = 2 * (stride * d - q * n); n2 = w.n2;
        i = first; iend = w.iend; S = stride;
        MS = stride * w.M + q * w.N; N = w.N;
        P = w.P;
    }
    LAMA_HD void step()
    {
        i += S;
        e2 += r2;
        P += (uint32_t)MS;
        if (e2 >= 0) { P += (uint32_t)N; e2 -= n2; }
    }
};

// Sector alignment of an x-major beam's strided segments: the delta in 0 .. 7 for which step 8 m + 1 - delta (m >= 1) is the first cell of an
// aligned octet of x in walk direction, x = 0 mod 8 when tx >= fx and x = 7 mod 8 when tx < fx (the major axis moves on every step).
// Window-relative x has the alignment of the cell's offset in its patch row, so the octet is one 32-byte sector of counters.
LAMA_HD int xmajor_seg_shift(uint32_t fx, uint32_t tx) { return (int)((tx < fx ? 0u - fx : fx + 1u) & 7u); }

// ---- event log ---------------------------------------------------------------------------------------
// log record: [cell key : 32][beam : 16][pos : 15][kind : 1], kind 1 = hit, 0 = miss.  Sorting the
// 64-bit records groups touches by cell and orders them by beam (a beam touches a cell at most once).
LAMA_HD uint64_t log_record(uint32_t key, uint32_t beam, uint32_t pos, bool hit)
{
    return ((uint64_t)key << 32) | ((uint64_t)(beam & 0xFFFFu) << 16) | ((uint64_t)(pos & 0x7FFFu) << 1) | (hit ? 1u : 0u);
}
LAMA_HD uint32_t log_key(uint64_t r) { return (uint32_t)(r >> 32); }
LAMA_HD uint32_t log_seq(uint64_t r) { return (uint32_t)r >> 1; }  // (beam << 15) | pos : the order of the reference's calls
LAMA_HD bool log_is_hit(uint64_t r) { return (r & 1u) != 0; }
// push record: [seq : 32][cell key : 32]; sorting by it orders obstacle events like the reference.
LAMA_HD uint64_t push_record(uint32_t seq, uint32_t key) { return ((uint64_t)seq << 32) | key; }

// Replays the sorted touches log[first, last) of ONE cell.  `word` is the occupancy word after all of this
// scan's atomics; it comes back with the carry of a wrapped `occupied` taken out (occ_drop_carry: every hit
// of the cell is in the log), and the caller stores it when it changed.  `obstacle` is the cell's
// obstacle-mirror bit before the scan; returns the new mirror bit and emits obstacle events through
// `emit(kind_is_add, seq)` in call order.
//   setFree     frequency_occupancy_map.cpp:65-74   setOccupied :81-91
//   addObstacle / removeObstacle no-op rules: dynamic_distance_map.cpp:217-218,233-234
template <typename Emit>
LAMA_HD bool replay_cell(const uint64_t* log, int first, int last, uint32_t& word, bool obstacle, Emit&& emit)
{
    uint32_t hits = 0, misses = 0;
    for (int i = first; i < last; ++i) {
        if (log_is_hit(log[i])) ++hits;
        else ++misses;
    }
    word = occ_drop_carry(word, hits);
    // counters before this scan (uint16 wrap-around arithmetic like the reference's cells)
    uint32_t occupied = (occ_occupied(word) - hits) & 0xFFFFu;
    uint32_t visited  = (occ_visited(word) - hits - misses) & 0xFFFFu;
    for (int i = first; i < last; ++i) {
        const uint64_t r = log[i];
        if (log_is_hit(r)) {
            bool was_occupied = occ_is_occupied(occupied, visited);
            occupied = (occupied + 1) & 0xFFFFu;
            visited  = (visited + 1) & 0xFFFFu;
            if (!was_occupied && occ_is_occupied(occupied, visited) && !obstacle) {
                obstacle = true;
                emit(true, log_seq(r));
            }
        } else {
            bool was_free = occ_is_free(occupied, visited);
            visited = (visited + 1) & 0xFFFFu;
            if (!was_free && occ_is_free(occupied, visited) && obstacle) {
                obstacle = false;
                emit(false, log_seq(r));
            }
        }
    }
    return obstacle;
}


// ---- ProbabilisticOccupancyMap (log-odds float cells) -------------------------------------------------------------
// src/sdm/probabilistic_occupancy_map.cpp:50-60 (constants), :82-91 setFree, :98-107 setOccupied.  The constants are
// computed on the host with the reference's float logods() and handed to the device as doubles.
struct ProbParams {
    double miss, hit, clamp_min, clamp_max, thresh;
};
LAMA_HD float prob_miss(float p, const ProbParams& pp) { return (float)fmax((double)p + pp.miss, pp.clamp_min); }
LAMA_HD float prob_hit(float p, const ProbParams& pp) { return (float)fmin((double)p + pp.hit, pp.clamp_max); }

// Ordered replay of the touches of one candidate cell of a log-odds map; returns the final cell value.
template <typename Emit>
LAMA_HD float replay_cell_prob(const uint64_t* log, int first, int last, float prob, bool& obstacle, const ProbParams& pp, Emit&& emit)
{
    for (int i = first; i < last; ++i) {
        const uint64_t r = log[i];
        if (log_is_hit(r)) {
            const bool was_occupied = (double)prob > pp.thresh;
            prob = prob_hit(prob, pp);
            if (!was_occupied && (double)prob > pp.thresh && !obstacle) {
                obstacle = true;
                emit(true, log_seq(r));
            }
        } else {
            const bool was_free = (double)prob < pp.thresh;
            prob = prob_miss(prob, pp);
            if (!was_free && (double)prob < pp.thresh && obstacle) {
                obstacle = false;
                emit(false, log_seq(r));
            }
        }
    }
    return prob;
}

}  // namespace lama_b200
