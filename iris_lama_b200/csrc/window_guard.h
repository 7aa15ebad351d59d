// window_guard.h -- where the directory window of a 2-D SLAM front end has to be before an update (Engine::shift_window moves it).
// Plain host C++; the CPU tests run it through tests/emu/window_shift_emu.cpp.
#pragma once

#include <algorithm>
#include <cmath>

#include "lama_core.h"

namespace lama_b200 {

// World AABB {mn, mx} of the endpoints of n points (xyz, sensor frame) seen from `pose` through the sensor transform m -- the transform
// the kernels apply (compose_tf) -- and of the sensor position.  *range = the largest distance of an endpoint from the pose's position.
inline void scan_guard_box(const SE2& pose, const MovingTf& m, const double* pts, int n, double mn[2], double mx[2], double* range)
{
    const Affine tf = compose_tf(pose, m);
    mn[0] = mx[0] = tf.t[0];
    mn[1] = mx[1] = tf.t[1];
    double r2 = (tf.t[0] - pose.tx) * (tf.t[0] - pose.tx) + (tf.t[1] - pose.ty) * (tf.t[1] - pose.ty);
    for (int i = 0; i < n; ++i) {
        double hit[3];
        apply_tf(tf, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], hit);
        for (int k = 0; k < 2; ++k) {
            mn[k] = std::min(mn[k], hit[k]);
            mx[k] = std::max(mx[k], hit[k]);
        }
        r2 = std::max(r2, (hit[0] - pose.tx) * (hit[0] - pose.tx) + (hit[1] - pose.ty) * (hit[1] - pose.ty));
    }
    *range = std::sqrt(r2);
}

// The guarded box of an update of `count` particles at predicted poses `poses`: the scan's box at poses[0], grown by the particles'
// spread (the diagonal of the box of their positions, plus their largest heading difference from poses[0] times the scan's range),
// by reach + 1 cells (the distance map's reach and the bilinear stencil) and by one patch of slack for the scan-match correction.
inline void guard_box(const SE2* poses, int count, const MovingTf& m, const double* pts, int n, double resolution, uint32_t reach_cells, double mn[2],
                      double mx[2])
{
    double range = 0.0;
    scan_guard_box(poses[0], m, pts, n, mn, mx, &range);
    double pmn[2] = {poses[0].tx, poses[0].ty}, pmx[2] = {poses[0].tx, poses[0].ty}, dth = 0.0;
    const double th0 = se2_rotation(poses[0]);
    for (int i = 1; i < count; ++i) {
        pmn[0] = std::min(pmn[0], poses[i].tx); pmx[0] = std::max(pmx[0], poses[i].tx);
        pmn[1] = std::min(pmn[1], poses[i].ty); pmx[1] = std::max(pmx[1], poses[i].ty);
        dth = std::max(dth, std::fabs(std::remainder(se2_rotation(poses[i]) - th0, 2 * M_PI)));
    }
    const double grow = std::hypot(pmx[0] - pmn[0], pmx[1] - pmn[1]) + dth * range + (double)(reach_cells + 1 + kPatchLen) * resolution;
    for (int k = 0; k < 2; ++k) {
        mn[k] -= grow;
        mx[k] += grow;
    }
}

enum : int { kGuardInside = 0, kGuardShift = 1, kGuardUnfit = 2 };

// The window's decision for a guarded world box {mn, mx} around a robot at world position `robot`: kGuardInside (every patch the box
// touches is in window w), kGuardShift (*base = the base of the window centred on the robot's patch, which holds the box) or kGuardUnfit
// (the window centred on the robot does not hold the box: the window stays, and the kernels report a touch outside it as they always
// do).  Centring on the robot rather than on the box keeps a few long beams from dragging the window away from where the robot is.
inline int window_guard(const DirWindow& w, const double mn[2], const double mx[2], const double robot[2], double scale, int32_t base[2])
{
    auto patch = [scale](double v) { return (int64_t)std::floor(v * scale + (double)kMapOffsetCells) >> kPatchLog2; };
    int64_t lo[2], hi[2], nb[2];
    for (int k = 0; k < 2; ++k) {
        lo[k] = patch(mn[k]);
        hi[k] = patch(mx[k]);
        nb[k] = patch(robot[k]) - w.dim / 2;
    }
    const int64_t cur[2] = {w.base_px, w.base_py};
    if (lo[0] >= cur[0] && hi[0] < cur[0] + w.dim && lo[1] >= cur[1] && hi[1] < cur[1] + w.dim) return kGuardInside;
    for (int k = 0; k < 2; ++k)
        if (nb[k] < 0 || lo[k] < nb[k] || hi[k] >= nb[k] + w.dim) return kGuardUnfit;
    base[0] = (int32_t)nb[0];
    base[1] = (int32_t)nb[1];
    return kGuardShift;
}

}  // namespace lama_b200
