"""A following DynamicDistanceMap on the CPU: the windows a following update runs its chunks in and the window of the dense directory
global localisation reads (iris_lama_b200/csrc/dm_follow.h, through the host build tests/emu/dm_follow_emu.cpp) against a plain Python
model, and the new C entry points."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATCH = 32
O = 1321122   # the patch of world 0 (kUniversalConstant / 2)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dm_follow_emu") / "libdm_follow_emu.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so,
                           os.path.join(HERE, "emu", "dm_follow_emu.cpp")])
    L = C.CDLL(so)
    L.emu_box_patches.restype = C.c_int64
    L.emu_brushfire_reach.restype = C.c_uint32
    return L


def plan(emu, base, dim, cells, chunk, reach):
    c = np.ascontiguousarray(np.asarray(cells, np.uint32).reshape(-1, 2))
    n_chunks = max(1, -(-len(c) // chunk))
    out = np.zeros(4 * n_chunks, np.int32)
    boxes = np.zeros((n_chunks, 4), np.int64)
    n = C.c_int(0)
    rc = emu.emu_plan_dm_chunks(C.c_int32(base[0]), C.c_int32(base[1]), C.c_int32(dim), c.ctypes.data_as(C.c_void_p), C.c_int(len(c)), C.c_int(chunk),
                                C.c_uint32(reach), out.ctypes.data_as(C.c_void_p), C.byref(n), boxes.ctypes.data_as(C.c_void_p))
    return rc, [tuple(int(v) for v in out[4 * i:4 * i + 4]) for i in range(n.value)], boxes


def extent(emu, mn, mx, n):
    out = np.zeros(3, np.int32)
    rc = emu.emu_extent_window(np.asarray(mn, np.uint32).ctypes.data_as(C.c_void_p), np.asarray(mx, np.uint32).ctypes.data_as(C.c_void_p), C.c_int(n),
                               out.ctypes.data_as(C.c_void_p))
    return rc, tuple(int(v) for v in out)


# ---- a plain model ----------------------------------------------------------------------------------------------------------------
def model_box(cells, reach):
    c = np.asarray(cells, np.int64).reshape(-1, 2)
    return (int(c[:, 0].min()) - reach, int(c[:, 1].min()) - reach, int(c[:, 0].max()) + reach, int(c[:, 1].max()) + reach)


def inside(base, dim, box):
    return all(base[k] <= box[k] // PATCH and box[2 + k] // PATCH < base[k] + dim for k in range(2))


def test_brushfire_reach_is_twice_the_map_reach(emu):
    # the reach a chunk's box is grown by: the brushfire writes within R of its cells and reads obstacles up to R further
    assert [emu.emu_brushfire_reach(r) for r in (1, 10, 20, 63)] == [2, 20, 40, 126]


def test_chunk_boxes_are_the_cells_grown_by_the_reach(emu):
    rng = np.random.default_rng(3)
    cells = (O * PATCH + rng.integers(-300, 300, (5000, 2))).astype(np.uint32)
    rc, groups, boxes = plan(emu, (O - 32, O - 32), 64, cells, 2048, 40)
    assert rc == -1 and len(boxes) == 3
    for k in range(3):
        assert tuple(boxes[k]) == model_box(cells[2048 * k:2048 * (k + 1)], 40), k
        assert emu.emu_box_patches(boxes[k].ctypes.data_as(C.c_void_p)) == \
            (boxes[k][2] // PATCH - boxes[k][0] // PATCH + 1) * (boxes[k][3] // PATCH - boxes[k][1] // PATCH + 1)
    assert groups == [(0, 3, O - 32, O - 32)]   # every box inside the current window: one group there, no shift


@pytest.mark.parametrize("side", range(4))
def test_boxes_on_the_window_edges(emu, side):
    dim, reach, base = 16, 40, (O - 8, O - 8)
    lo, hi = base[0] * PATCH, (base[0] + dim) * PATCH - 1   # first and last cell of the window on each axis
    mid = (lo + hi) // 2
    # a cell whose grown box ends exactly on the window's first / last cell stays; one cell further moves the window
    edge = [(lo + reach, mid), (hi - reach, mid), (mid, lo + reach), (mid, hi - reach)][side]
    out = [(lo + reach - 1, mid), (hi - reach + 1, mid), (mid, lo + reach - 1), (mid, hi - reach + 1)][side]
    rc, groups, _ = plan(emu, base, dim, [edge], 2048, reach)
    assert rc == -1 and groups == [(0, 1, base[0], base[1])]
    rc, groups, boxes = plan(emu, base, dim, [out], 2048, reach)
    assert rc == -1 and len(groups) == 1 and (groups[0][2], groups[0][3]) != base
    assert inside(groups[0][2:], dim, boxes[0])


def test_a_chunk_wider_than_a_window_is_refused_before_any_group(emu):
    dim, reach, base = 8, 20, (O - 4, O - 4)
    c0 = O * PATCH
    ok = [(c0, c0)] * 2048
    # chunk 1 spans exactly dim patches once grown (fits), chunk 2 one cell more (dim + 1 patches)
    fits = [(c0 - (dim * PATCH) // 2 + reach, c0), (c0 + (dim * PATCH) // 2 - 1 - reach, c0)] * 1024
    wide = [(c0 - (dim * PATCH) // 2 + reach, c0), (c0 + (dim * PATCH) // 2 - reach, c0)] * 1024
    rc, groups, _ = plan(emu, base, dim, ok + fits, 2048, reach)
    assert rc == -1 and sum(g[1] for g in groups) == 2
    rc, groups, _ = plan(emu, base, dim, ok + fits + wide, 2048, reach)
    assert rc == 2 and groups == []


def test_random_updates_split_into_ordered_groups_whose_windows_hold_their_chunks(emu):
    rng = np.random.default_rng(7)
    dim, reach, chunk = 16, 20, 64
    for trial in range(30):
        n = int(rng.integers(1, 1500))
        walk = np.cumsum(rng.integers(-40, 41, (n, 2)), axis=0) + O * PATCH
        cells = (walk + rng.integers(-30, 31, (n, 2))).astype(np.uint32)
        rc, groups, boxes = plan(emu, (O - 8, O - 8), dim, cells, chunk, reach)
        if rc >= 0:   # refused: that chunk's box is wider than a window
            b = model_box(cells[chunk * rc:chunk * (rc + 1)], reach)
            assert max(b[2] // PATCH - b[0] // PATCH, b[3] // PATCH - b[1] // PATCH) + 1 > dim and groups == []
            continue
        assert groups[0][0] == 0 and sum(g[1] for g in groups) == len(boxes)
        for a, b in zip(groups, groups[1:]):
            assert b[0] == a[0] + a[1] and (b[2], b[3]) != (a[2], a[3])
            assert not inside(a[2:], dim, boxes[b[0]])   # a new window opens only when the current one misses the next chunk
        for first, count, bx, by in groups:
            for k in range(first, first + count):
                assert inside((bx, by), dim, boxes[k]), (trial, k)


def test_extent_window_of_the_map_bounds(emu):
    cap = emu.emu_extent_cap()
    assert cap == 4096
    assert extent(emu, (0, 0), (0, 0), 0)[0] == 0                       # an empty map: nothing to build
    b = O * PATCH
    rc, w = extent(emu, (b, b - 64), (b + 10 * PATCH, b + 3 * PATCH), 12)   # 10 x 5 patches: a square of the larger span
    assert rc == 1 and w == (O, O - 2, 10)
    rc, w = extent(emu, (b, b), (b + cap * PATCH, b + PATCH), 5)         # exactly the cap
    assert rc == 1 and w == (O, O, cap)
    assert extent(emu, (b, b), (b + PATCH, b + (cap + 1) * PATCH), 5)[0] == -1   # one patch more on either axis
    assert extent(emu, (b, b), (b + (cap + 1) * PATCH, b + PATCH), 5)[0] == -1


# ---- C-ABI ------------------------------------------------------------------------------------------------------------------------
NEW = ["lama_dm_set_follow", "lama_dm_get_window", "lama_dm_get_pool", "lama_dm_kernel_times"]


def test_new_entry_points_are_declared_and_exported(api):
    src = open(os.path.join(ROOT, "include", "lama_b200.h")).read()
    L = api.lib()
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, src) and n in api.EXPORTED_SYMBOLS and hasattr(L, n), n


def test_new_entry_points_refuse_null_handles_and_outputs(api):
    L = api.lib()
    null = C.c_void_p(None)
    b2 = (C.c_int32 * 2)()
    d = C.c_int32(0)
    c3 = (C.c_uint64 * 3)()
    ms, ln = (C.c_double * 4)(), (C.c_uint64 * 5)()
    for fn, args in [(L.lama_dm_set_follow, (null, C.c_int(1))), (L.lama_dm_get_window, (null, b2, C.byref(d), c3)),
                     (L.lama_dm_get_pool, (null, c3)), (L.lama_dm_kernel_times, (null, ms, ln))]:
        fn.restype = C.c_int
        L.lama_last_error.restype = C.c_char_p
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0, fn.__name__
    if api.device_count() > 0:   # null outputs on a live map
        m = api.DynamicDistanceMap(0.05, follow=True)
        assert L.lama_dm_get_window(m.h, None, C.byref(d), c3) == -1 and len(L.lama_last_error()) > 0
        assert L.lama_dm_get_pool(m.h, None) == -1 and len(L.lama_last_error()) > 0


def test_following_distance_map_needs_a_gpu_or_fails_loudly(api):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.LamaError) as e:
        api.DynamicDistanceMap(0.05, follow=True)
    assert e.value.code == -3


def test_shim_caller_that_sets_follow_compiles(tmp_path):
    src = tmp_path / "shim.cpp"
    src.write_text('#include "lama_b200_shim.hpp"\nint main() { lama_dm* m = nullptr; lama_b200_shim::Loc2D* loc = nullptr;\n'
                   ' if (m) { lama_b200_shim::distanceMapSetFollow(m, true); auto w = lama_b200_shim::distanceMapWindow(m); uint64_t p[2];\n'
                   ' lama_b200_shim::distanceMapPool(m, p); return (int)w.dim; }\n'
                   ' if (loc) { loc->setFollow(true); loc->readDistanceMap("map.sdm"); return (int)loc->window().parked; }\n'
                   ' return 0; }\n')
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])
