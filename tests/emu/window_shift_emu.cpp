// Test-only host build of window_shift_core.h and window_guard.h: the window shift as k_shift_count / k_shift_apply run it (the same
// per-entry functions, the prefix sums computed serially), and the window guard's decision.
#include <cstdint>
#include <vector>

#include "../../iris_lama_b200/csrc/window_guard.h"
#include "../../iris_lama_b200/csrc/window_shift_core.h"

using namespace lama_b200;

extern "C" {

// Shifts one map (directory `dir` of window {base_px, base_py, dim}, parked list of n_parked entries as px, py, entry triples) to base
// (nbx, nby).  dir is rewritten in place; the new list goes to out_parked (room for n_parked + dim^2 entries).  Returns its length.
int emu_shift(int32_t base_px, int32_t base_py, int32_t dim, int32_t nbx, int32_t nby, int32_t* dir, const int32_t* parked, int n_parked,
              int32_t* out_parked, int* entered)
{
    const DirWindow w{base_px, base_py, dim}, nw{nbx, nby, dim};
    const int dim2 = dim * dim;
    const ParkEntry* A = reinterpret_cast<const ParkEntry*>(parked);
    std::vector<int32_t> od(dir, dir + dim2), leave_before(dim2 + 1), enter_before(n_parked + 1);
    int leave = 0, enter = 0;
    for (int i = 0; i < dim2; ++i) { leave_before[i] = leave; leave += shift_leaves(w, nw, i, od[i]) ? 1 : 0; }
    leave_before[dim2] = leave;
    for (int i = 0; i < n_parked; ++i) { enter_before[i] = enter; enter += shift_enters(nw, A[i]) ? 1 : 0; }
    enter_before[n_parked] = enter;
    for (int j = 0; j < dim2; ++j) dir[j] = shift_new_entry(w, nw, j, od.data(), A, n_parked);
    ParkEntry* C = reinterpret_cast<ParkEntry*>(out_parked);
    for (int i = 0; i < n_parked; ++i)
        if (!shift_enters(nw, A[i])) C[shift_pos_parked(w, A, i, enter_before.data(), leave_before.data())] = A[i];
    for (int i = 0; i < dim2; ++i)
        if (shift_leaves(w, nw, i, od[i])) {
            ParkEntry e{w.base_px + i % dim, w.base_py + i / dim, od[i]};
            C[shift_pos_leaving(w, i, A, n_parked, enter_before.data(), leave_before.data())] = e;
        }
    *entered = enter;
    return n_parked - enter + leave;
}

// k_shift_apply's scratch writes for lists ol ({offset, length} pairs) into a buffer of shift_scratch_ints: 0 when every write of every
// list lands inside it and no two lists overlap, else 1
int emu_shift_scratch_check(const int32_t* ol, int n_lists)
{
    std::vector<int> hits(shift_scratch_ints(ol, n_lists), 0);
    for (int i = 0; i < n_lists; ++i)
        for (int k = 0; k <= ol[2 * i + 1]; ++k) {
            const size_t at = (size_t)shift_enter_base(ol[2 * i], i) + k;
            if (at >= hits.size() || hits[at]++) return 1;
        }
    return 0;
}

int32_t emu_park_find(const int32_t* parked, int n, int32_t px, int32_t py)
{
    return park_find(reinterpret_cast<const ParkEntry*>(parked), n, px, py);
}

// window_guard for the world box {mn, mx} around a robot at `robot`, at 1 / scale m per cell
int emu_window_guard(int32_t base_px, int32_t base_py, int32_t dim, const double* mn, const double* mx, const double* robot, double scale, int32_t* base)
{
    return window_guard(DirWindow{base_px, base_py, dim}, mn, mx, robot, scale, base);
}

// guard_box of `count` poses (x, y, theta) and n points (xyz) through an identity sensor transform
void emu_guard_box(const double* xyr, int count, const double* pts, int n, double resolution, uint32_t reach, double* mn, double* mx)
{
    std::vector<SE2> poses((size_t)count);
    for (int i = 0; i < count; ++i) poses[i] = se2_from_xyr(xyr[3 * i], xyr[3 * i + 1], xyr[3 * i + 2]);
    MovingTf m{};
    m.l[0] = m.l[4] = m.l[8] = 1.0;
    guard_box(poses.data(), count, m, pts, n, resolution, reach, mn, mx);
}

}  // extern "C"
