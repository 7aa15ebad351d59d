// lama_core.h -- cell encodings, grid addressing and SE2 algebra shared by the sm_90a kernels and
// the host engine.  Everything here is plain C++ usable from both host and device code.
//
// Reference behaviour being reproduced (paths relative to the reference tree):
//   grid addressing   include/lama/sdm/map.h:125-189, src/sdm/map.cpp:42-58
//   frequency cell    include/lama/sdm/frequency_occupancy_map.h:43-46, src/sdm/frequency_occupancy_map.cpp:38-91
//   distance cell     include/lama/sdm/dynamic_distance_map.h:48-53
//   SE2 / SO2         include/lama/sophus/so2.hpp:167-214,246-278,322-324,401-404, se2.hpp:153-168,233-265,389-412
#pragma once

#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define LAMA_HD __host__ __device__ __forceinline__
#else
#define LAMA_HD inline
#endif

namespace lama_b200 {

// ------------------------------------------------------------------------------------------------
// Device data layout.
//
// A map (occupancy or distance) of one particle is a dense DIRECTORY of patch slots covering a
// square window of dir_dim x dir_dim patches, plus 4 KiB patches (32 x 32 cells x 4 B) living in a
// pool shared by all particles and both map kinds.  Patches are reference counted and shared
// copy-on-write between particles (the reference's COWPtr<Container>, cow_ptr.h:96-114).
// ------------------------------------------------------------------------------------------------
constexpr int kPatchLog2   = 5;
constexpr int kPatchLen    = 1 << kPatchLog2;        // 32 cells (Options::patch_size default)
constexpr int kPatchCells  = kPatchLen * kPatchLen;  // 1024
constexpr int kPatchBytes  = kPatchCells * 4;        // 4096
constexpr uint32_t kUniversalHalf = 1321122u;        // UNIVERSAL_CONSTANT >> 1 (map.h:68, map.cpp:55)
constexpr uint32_t kMapOffsetCells = kUniversalHalf * kPatchLen;  // 42 275 904

// ---- occupancy cell: FrequencyOccupancyMap {uint16 occupied; uint16 visited} packed in one word so
// that a hit is ONE atomicAdd(+0x00010001) and a miss ONE atomicAdd(+0x00010000); `visited` (high half)
// wraps at 2^16 exactly like the reference's uint16.  The reference's two counters are independent, but in the
// packed word the 65 536th hit of a cell carries out of `occupied` into `visited`: every writer that adds hits
// takes that carry back (occ_drop_carry in the ray-cast replay, a returning add in the render).
// Whether a cell is currently an obstacle of the distance map (valid_obstacle && sqdist == 0) -- which
// decides if a miss can trigger removeObstacle -- is mirrored in a separate bit plane of 32 words per patch
// (StoreView::fbits), so that the ray-cast kernel never needs the value returned by an atomic.
constexpr uint32_t kOccHitInc   = 0x00010001u;
constexpr uint32_t kOccMissInc  = 0x00010000u;
LAMA_HD uint32_t occ_occupied(uint32_t w) { return w & 0xFFFFu; }
LAMA_HD uint32_t occ_visited(uint32_t w) { return w >> 16; }
// `word` after `hits` (< 2^16) packed hits and any number of misses: `occupied` carried into `visited` at most once, and it did
// exactly when the final `occupied` is below `hits`.  Returns the word with that carry taken back.
LAMA_HD uint32_t occ_drop_carry(uint32_t word, uint32_t hits) { return occ_occupied(word) < hits ? word - kOccMissInc : word; }
// prob() < 0.25 / > 0.25 of frequency_occupancy_map.cpp:40-45 in exact integer arithmetic
// (occupied/visited == 0.25 exactly iff 4*occupied == visited; unvisited cells read 0.25).
LAMA_HD bool occ_is_free(uint32_t occupied, uint32_t visited) { return visited != 0 && 4u * occupied < visited; }
LAMA_HD bool occ_is_occupied(uint32_t occupied, uint32_t visited) { return visited != 0 && 4u * occupied > visited; }

// ---- distance cell: DynamicDistanceMap::distance_t {int16 obstacle[3]; uint16 sqdist; bool valid;
// bool queued} packed into one word: sqdist 12 bits, 7-bit two's complement x / y offsets, flags.
// This bounds the truncation radius to 63 cells (l2_max * scale <= 63); the 2-D front ends use 10
// (PFSlam2D/Slam2D, l2_max 0.5 m) and 20 (Loc2D, l2_max 1.0 m) cells.
constexpr uint32_t kDmSqMask   = 0x00000FFFu;
constexpr int      kDmOxShift  = 12;
constexpr int      kDmOyShift  = 19;
constexpr uint32_t kDmValid    = 1u << 26;
constexpr uint32_t kDmQueued   = 1u << 27;
constexpr uint32_t kDmKnown    = 1u << 28;   // Container bitmask bit (container.h:102-123)
constexpr int      kDmMaxRadius = 63;
LAMA_HD uint32_t dm_sqdist(uint32_t w) { return w & kDmSqMask; }
LAMA_HD int dm_ox(uint32_t w) { return (int)(w << (32 - kDmOxShift - 7)) >> 25; }
LAMA_HD int dm_oy(uint32_t w) { return (int)(w << (32 - kDmOyShift - 7)) >> 25; }
LAMA_HD uint32_t dm_pack(uint32_t sqdist, int ox, int oy, bool valid, bool queued)
{
    return (sqdist & kDmSqMask) | (((uint32_t)ox & 0x7Fu) << kDmOxShift) | (((uint32_t)oy & 0x7Fu) << kDmOyShift) |
           (valid ? kDmValid : 0u) | (queued ? kDmQueued : 0u) | kDmKnown;
}

// ---- directory window -----------------------------------------------------------------------------
struct DirWindow {
    int32_t base_px, base_py;  // patch coordinates (cell >> 5) of directory entry (0,0)
    int32_t dim;               // entries per side (power of two)
};
// a directory entry is -1 or slot | flags (the flags are described in device_store.cuh)
constexpr int32_t kDirSlotMask = 0x00FFFFFF;
constexpr int32_t kDirHot      = 1 << 28;
constexpr int32_t kDirOwn      = 1 << 29;
// directory index of the patch holding cell (x, y), or -1 when outside the window.
LAMA_HD int dir_index(const DirWindow& w, uint32_t x, uint32_t y)
{
    int px = (int)(x >> kPatchLog2) - w.base_px, py = (int)(y >> kPatchLog2) - w.base_py;
    if ((unsigned)px >= (unsigned)w.dim || (unsigned)py >= (unsigned)w.dim) return -1;
    return py * w.dim + px;
}
// cell index inside the patch: (x & 31) | ((y & 31) << 5)  (map.h:182-189)
LAMA_HD uint32_t cell_index(uint32_t x, uint32_t y) { return (x & (kPatchLen - 1)) | ((y & (kPatchLen - 1)) << kPatchLog2); }
// window-relative 32-bit cell key used by logs, heaps and hash sets: y_rel << 16 | x_rel
LAMA_HD uint32_t cell_key(const DirWindow& w, uint32_t x, uint32_t y)
{
    return ((y - ((uint32_t)w.base_py << kPatchLog2)) << 16) | ((x - ((uint32_t)w.base_px << kPatchLog2)) & 0xFFFFu);
}
LAMA_HD uint32_t key_x(const DirWindow& w, uint32_t key) { return (key & 0xFFFFu) + ((uint32_t)w.base_px << kPatchLog2); }
LAMA_HD uint32_t key_y(const DirWindow& w, uint32_t key) { return (key >> 16) + ((uint32_t)w.base_py << kPatchLog2); }

// ---- exact-rounding arithmetic helpers ---------------------------------------------------------------
// World -> map coordinates must round exactly like the reference's `p * scale + offset`
// (map.h:125-138) with no fused multiply-add, otherwise an endpoint can land in another cell.
#if defined(__CUDA_ARCH__)
LAMA_HD double mul_rn(double a, double b) { return __dmul_rn(a, b); }
LAMA_HD double add_rn(double a, double b) { return __dadd_rn(a, b); }
#else
LAMA_HD double mul_rn(double a, double b) { volatile double r = a * b; return r; }
LAMA_HD double add_rn(double a, double b) { volatile double r = a + b; return r; }
#endif

LAMA_HD double w2m_nocast(double p, double scale) { return add_rn(mul_rn(p, scale), (double)kMapOffsetCells); }  // map.h:137
LAMA_HD uint32_t w2m(double p, double scale) { return (uint32_t)add_rn(w2m_nocast(p, scale), 0.5); }            // map.h:125-126

// ---- SE2 -----------------------------------------------------------------------------------------------
struct SE2 {
    double c, s, tx, ty;
};
constexpr double kLieEps = 1e-10;  // sophus.hpp:37-39

LAMA_HD void so2_normalize(double& c, double& s)  // so2.hpp:246-255 (the zero-norm exception cannot trigger here)
{
    double len = sqrt(add_rn(mul_rn(c, c), mul_rn(s, s)));
    c /= len;
    s /= len;
}
LAMA_HD SE2 se2_mul(const SE2& a, const SE2& b)  // se2.hpp:153-157,262-265 ; so2.hpp:167-176,275-278
{
    SE2 r;
    r.tx = add_rn(a.tx, add_rn(mul_rn(a.c, b.tx), -mul_rn(a.s, b.ty)));
    r.ty = add_rn(a.ty, add_rn(mul_rn(a.s, b.tx), mul_rn(a.c, b.ty)));
    r.c  = add_rn(mul_rn(a.c, b.c), -mul_rn(a.s, b.s));
    r.s  = add_rn(mul_rn(a.c, b.s), mul_rn(a.s, b.c));
    so2_normalize(r.c, r.s);
    return r;
}
LAMA_HD SE2 se2_exp(const double h[3])  // se2.hpp:389-412
{
    double theta = h[2];
    SE2 r;
    r.c = cos(theta);
    r.s = sin(theta);
    so2_normalize(r.c, r.s);
    double a, b;
    if (fabs(theta) < kLieEps) {
        double theta_sq = mul_rn(theta, theta);
        a = add_rn(1., -mul_rn(1. / 6., theta_sq));
        b = add_rn(mul_rn(0.5, theta), -mul_rn(mul_rn(1. / 24., theta), theta_sq));
    } else {
        a = r.s / theta;
        b = add_rn(1., -r.c) / theta;
    }
    r.tx = add_rn(mul_rn(a, h[0]), -mul_rn(b, h[1]));
    r.ty = add_rn(mul_rn(b, h[0]), mul_rn(a, h[1]));
    return r;
}
LAMA_HD SE2 se2_inv(const SE2& a)  // se2.hpp:163-167 ; so2.hpp:192-194
{
    SE2 r;
    r.c = a.c;
    r.s = -a.s;
    so2_normalize(r.c, r.s);
    double nx = mul_rn(a.tx, -1.0), ny = mul_rn(a.ty, -1.0);
    r.tx = add_rn(mul_rn(r.c, nx), -mul_rn(r.s, ny));
    r.ty = add_rn(mul_rn(r.s, nx), mul_rn(r.c, ny));
    return r;
}
LAMA_HD SE2 se2_from_xyr(double x, double y, double theta)  // se2.hpp:648-651
{
    SE2 r;
    r.c = cos(theta);
    r.s = sin(theta);
    so2_normalize(r.c, r.s);
    r.tx = x;
    r.ty = y;
    return r;
}
LAMA_HD double se2_rotation(const SE2& a) { return atan2(a.s, a.c); }  // so2.hpp:401-404
// SE2::log (se2.hpp:519-542): (upsilon, theta) with upsilon = V^-1 t
LAMA_HD void se2_log(const SE2& a, double out[3])
{
    const double theta = se2_rotation(a), half = 0.5 * theta;
    const double real_minus_one = a.c - 1.0;
    double h;
    if (fabs(real_minus_one) < kLieEps) h = 1.0 - (1.0 / 12.0) * theta * theta;
    else h = -(half * a.s) / real_minus_one;
    out[0] = h * a.tx + half * a.ty;
    out[1] = -half * a.tx + h * a.ty;
    out[2] = theta;
}
// SE2::Adj (se2.hpp:125-133), row major 3 x 3
LAMA_HD void se2_adj(const SE2& a, double m[9])
{
    m[0] = a.c; m[1] = -a.s; m[2] = a.ty;
    m[3] = a.s; m[4] = a.c;  m[5] = -a.tx;
    m[6] = 0.0; m[7] = 0.0;  m[8] = 1.0;
}

// ---- sensor -> map transform ---------------------------------------------------------------------------
// tf = [T(x,y,0) Rz(theta)] * [T(sensor_origin) R(sensor_quat)]   (match_surface_2d.cpp:49-58,
// pf_slam2d.cpp:397-403,444-452).  The moving part is constant per scan and prepared on the host
// (ScanTf::ml / mt); the fixed part changes with the particle pose.
struct MovingTf {
    double l[9];  // row-major rotation of the sensor
    double t[3];  // sensor origin
};
struct Affine {
    double l[9];
    double t[3];
};
LAMA_HD Affine compose_tf(const SE2& pose, const MovingTf& m)
{
    // Rz is rebuilt from theta = atan2(s, c) exactly like AngleAxisd(state.so2().log(), UnitZ).
    const double theta = se2_rotation(pose);
    const double s = sin(theta), c = cos(theta);
    const double f[9] = {c, -s, 0, s, c, 0, 0, 0, add_rn(add_rn(1, -c), c)};
    const double ft[3] = {pose.tx, pose.ty, 0.0};
    Affine r;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            r.l[i * 3 + j] = add_rn(add_rn(mul_rn(f[i * 3 + 0], m.l[0 * 3 + j]), mul_rn(f[i * 3 + 1], m.l[1 * 3 + j])), mul_rn(f[i * 3 + 2], m.l[2 * 3 + j]));
        r.t[i] = add_rn(add_rn(add_rn(mul_rn(f[i * 3 + 0], m.t[0]), mul_rn(f[i * 3 + 1], m.t[1])), mul_rn(f[i * 3 + 2], m.t[2])), ft[i]);
    }
    return r;
}
// The same transform with Rz built straight from the unit complex number of the state: cos(atan2(s, c)) and c differ by a few
// 1e-16, so this is the transform of compose_tf up to the last bits -- good for the residual evaluations of the scan matcher (sums
// reduced in another order than the reference's anyway), NOT for the map update, where a last-bit difference can move a hit cell.
LAMA_HD Affine compose_tf_fast(const SE2& pose, const MovingTf& m)
{
    const double s = pose.s, c = pose.c;
    const double f[9] = {c, -s, 0, s, c, 0, 0, 0, 1.0};
    const double ft[3] = {pose.tx, pose.ty, 0.0};
    Affine r;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            r.l[i * 3 + j] = add_rn(add_rn(mul_rn(f[i * 3 + 0], m.l[0 * 3 + j]), mul_rn(f[i * 3 + 1], m.l[1 * 3 + j])), mul_rn(f[i * 3 + 2], m.l[2 * 3 + j]));
        r.t[i] = add_rn(add_rn(add_rn(mul_rn(f[i * 3 + 0], m.t[0]), mul_rn(f[i * 3 + 1], m.t[1])), mul_rn(f[i * 3 + 2], m.t[2])), ft[i]);
    }
    return r;
}
LAMA_HD void apply_tf(const Affine& a, double px, double py, double pz, double out[3])
{
    for (int i = 0; i < 3; ++i)
        out[i] = add_rn(add_rn(add_rn(mul_rn(a.l[i * 3 + 0], px), mul_rn(a.l[i * 3 + 1], py)), mul_rn(a.l[i * 3 + 2], pz)), a.t[i]);
}

// error bits accumulated in the per-handle device status word
enum : uint32_t {
    kErrWindow       = 1u << 0,  // a cell outside the directory window was addressed
    kErrPoolEmpty    = 1u << 1,  // the patch pool ran out of slots
    kErrEventLog     = 1u << 2,  // per-scan event log overflow (ray-cast kernel)
    kErrHeapOverflow = 1u << 3,  // brushfire heap overflow
    kErrPushOverflow = 1u << 4,  // obstacle add/remove list overflow
};

}  // namespace lama_b200
