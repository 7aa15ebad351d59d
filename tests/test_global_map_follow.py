"""A global map without an edge, on the CPU: the render plan and the pool growth of a following FrequencyOccupancyMap
(iris_lama_b200/csrc/render_plan.h, through the host build tests/emu/render_plan_emu.cpp) against a plain Python model; kind-4 checkpoints
whose global map has parked entries and a grown pool, from an independent writer; and the new C entry points."""
import ctypes as C
import os
import re
import struct
import subprocess

import numpy as np
import pytest

from test_checkpoint import frame
import test_graph_checkpoint as tg

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATCH = 32
CAP = (1 << 24) - 2
O = 1321122   # the patch of world 0 (kUniversalConstant / 2)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("render_plan_emu") / "librender_plan_emu.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so,
                           os.path.join(HERE, "emu", "render_plan_emu.cpp")])
    L = C.CDLL(so)
    L.emu_pool_growth.restype = C.c_int64
    L.emu_pool_growth.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int]
    return L


def plan(emu, base, dim, boxes):
    b = np.ascontiguousarray(np.asarray(boxes, np.int64).reshape(-1, 4))
    out = np.zeros(4 * max(1, len(b)), np.int32)
    n = C.c_int(0)
    rc = emu.emu_plan_render(C.c_int32(base[0]), C.c_int32(base[1]), C.c_int32(dim), b.ctypes.data_as(C.c_void_p), C.c_int(len(b)),
                             out.ctypes.data_as(C.c_void_p), C.byref(n))
    return rc, [tuple(int(v) for v in out[4 * i:4 * i + 4]) for i in range(n.value)]


# ---- a plain model ----------------------------------------------------------------------------------------------------------------
def inside(base, dim, box):
    return all(base[k] <= box[k] // PATCH and box[2 + k] // PATCH < base[k] + dim for k in range(2))


def fits_some_window(dim, box):
    return all(box[2 + k] // PATCH - box[k] // PATCH + 1 <= dim for k in range(2))


def random_boxes(rng, n, dim, step, width):
    """n scans along a random walk of `step` cells per scan, boxes up to `width` cells wide"""
    c = np.array([O * PATCH, O * PATCH], np.int64)
    out = []
    for _ in range(n):
        c += rng.integers(-step, step + 1, 2)
        w = rng.integers(1, width + 1, 2)
        lo = c - rng.integers(0, w + 1)
        out.append((int(lo[0]), int(lo[1]), int(lo[0] + w[0]), int(lo[1] + w[1])))
    return out


@pytest.mark.parametrize("dim", [8, 16, 64])
def test_random_sequences_split_into_ordered_groups_whose_windows_hold_their_scans(emu, dim):
    rng = np.random.default_rng(dim)
    base = (O - dim // 2, O - dim // 2)
    for trial in range(40):
        boxes = random_boxes(rng, int(rng.integers(1, 120)), dim, int(rng.integers(1, dim * PATCH // 2)), dim * PATCH - 2 * PATCH)
        rc, groups = plan(emu, base, dim, boxes)
        assert rc == -1
        # every scan in exactly one group, in order
        assert groups[0][0] == 0 and sum(g[1] for g in groups) == len(boxes)
        for a, b in zip(groups, groups[1:]):
            assert b[0] == a[0] + a[1]
        cur = base
        for first, count, bx, by in groups:
            w = (bx, by)
            for k in range(first, first + count):   # every box inside its group's window, patch-aligned by construction
                assert inside(w, dim, boxes[k])
            if first > 0:   # a group starts only where the scan leaves the previous window
                assert not inside(cur, dim, boxes[first]) and w != cur
                # the new window is centred on that scan's box (to half a patch)
                for k in range(2):
                    lo, hi = boxes[first][k] // PATCH, boxes[first][2 + k] // PATCH
                    assert abs((lo - w[k]) - (w[k] + dim - 1 - hi)) <= 1
            elif w != base:
                assert not inside(base, dim, boxes[0])
            cur = w


def test_scans_that_fit_the_current_window_make_one_group_and_no_shift(emu):
    dim = 16
    base = (O - 8, O - 8)
    rng = np.random.default_rng(5)
    lo = np.array(base) * PATCH
    for _ in range(20):
        boxes = []
        for _ in range(int(rng.integers(1, 50))):
            a = lo + rng.integers(0, dim * PATCH - 40, 2)
            boxes.append((int(a[0]), int(a[1]), int(a[0] + rng.integers(0, 39)), int(a[1] + rng.integers(0, 39))))
        rc, groups = plan(emu, base, dim, boxes)
        assert rc == -1 and groups == [(0, len(boxes), base[0], base[1])]


def test_a_scan_wider_than_the_window_is_refused_with_its_index_before_any_group(emu):
    dim = 8
    base = (O - 4, O - 4)
    c = O * PATCH
    ok = (c, c, c + 10, c + 10)
    far = (c + 5000, c, c + 5010, c + 10)          # fits a window, elsewhere
    wide = (c, c, c + dim * PATCH, c + 10)          # dim * 32 + 1 cells: no window holds it
    straddle = (c + 16, c, c + 16 + dim * PATCH - 1, c + 10)   # dim * 32 cells across dim + 1 patches
    tall = (c, c - 1000, c + 10, c + dim * PATCH)
    for boxes, bad in [([ok, far, wide], 2), ([wide], 0), ([ok, straddle, far], 1), ([far, ok, ok, tall], 3)]:
        rc, groups = plan(emu, base, dim, boxes)
        assert rc == bad and groups == []
    # the widest box that fits: exactly dim patches
    rc, groups = plan(emu, base, dim, [(c, c, c + dim * PATCH - 1, c + 10)])
    assert rc == -1 and len(groups) == 1 and groups[0][2] == O


def test_scan_box_holds_the_hits_and_the_ray_start_with_one_cell_of_slack(emu):
    pts = np.array([[3.0, 0.0, 0.0], [-1.0, 2.0, 0.0], [0.5, -4.0, 0.0]])
    out = np.zeros(4, np.int64)
    emu.emu_render_scan_box((C.c_double * 3)(1.0, -2.0, 0.0), pts.ctypes.data_as(C.c_void_p), C.c_int(3), C.c_double(20.0),
                            out.ctypes.data_as(C.c_void_p))
    xs = np.array([1.0, 4.0, 0.0, 1.5]) * 20 + O * PATCH
    ys = np.array([-2.0, -2.0, 0.0, -6.0]) * 20 + O * PATCH
    assert out.tolist() == [int(np.floor(xs.min() + 0.5)) - 1, int(np.floor(ys.min() + 0.5)) - 1, int(np.floor(xs.max() + 0.5)) + 1,
                            int(np.floor(ys.max() + 0.5)) + 1]


def model_growth(n, held, dim2, growable):
    """held: slots held outside the window (parked)"""
    if not growable or n - held >= dim2 or n >= CAP:
        return n
    while n < held + dim2:
        n *= 2
    return min(n, CAP)


def test_pool_growth_doubles_to_hold_the_parked_patches_and_a_window_and_stops_at_the_slot_cap(emu):
    g = emu.emu_pool_growth
    assert g(256, 0, 256, 1) == 256                  # a dir_dim^2 pool holds a whole window: a map that never moves never grows
    assert g(256, 1, 256, 1) == 512
    assert g(256, 200, 256, 1) == 512
    assert g(256, 256, 256, 1) == 512
    assert g(4096, 4000, 4096, 1) == 8192
    assert g(1024, 1000, 4096, 1) == 8192            # doubled until parked + dim^2 fit
    assert g(1 << 23, (1 << 23) - 10, 4096, 1) == CAP  # capped at 2^24 - 2
    assert g(CAP, CAP - 1, 4096, 1) == CAP
    assert g(300, 299, 256, 0) == 300                # an explicit pool never grows
    rng = np.random.default_rng(1)
    for _ in range(2000):
        dim2 = int(rng.choice([64, 256, 1024, 4096, 16384]))
        n = int(rng.integers(dim2, 1 << 24))
        held = int(rng.integers(0, n + 1))
        grow = int(rng.integers(0, 2))
        m = g(n, held, dim2, grow)
        assert m == model_growth(n, held, dim2, grow)
        assert n <= m <= max(n, CAP)
        if m != n:   # the smallest doubling of n that holds the parked slots and a window, or the cap
            assert grow and (m == CAP or (m % n == 0 and m >= held + dim2 and m // 2 < held + dim2))


# ---- kind-4 checkpoints with a parked, grown global map ---------------------------------------------------------------------------
MARKER = b"LAMAPARK"
DIM = 8
BASE = O - DIM // 2
FAR = BASE + 40
KNOWN_STRIDE = 4096 + 128 + 128


def engine_v2(pool, known_plane, lists, refcount, dir_entries, res=0.05, l2=0.5):
    """a version-2 engine section (one particle, frequency map) and its slots: dir_entries {(kind, index): entry}, lists
    {(kind): [(px, py, entry), ...]} parked between the directories and the slots"""
    K = len(refcount)
    b = b"\x01" + struct.pack("<5i", 1, DIM, pool, 2048, 0) + bytes([1 if known_plane else 0])
    b += struct.pack("<2d", res, l2) + struct.pack("<2i", BASE, BASE)
    b += struct.pack("<3QI", K, 0, 0, K) + struct.pack(f"<{K}i", *refcount)
    dirs = np.full((1, 2, DIM * DIM), -1, np.int32)
    for (k, i), e in dir_entries.items():
        dirs[0, k, i] = e
    b += dirs.tobytes()
    b += struct.pack("<2I", *(len(lists.get(k, [])) for k in range(2)))
    for k in range(2):
        for e in lists.get(k, []):
            b += struct.pack("<3i", *e)
    stride = 4096 + 128 + (128 if known_plane else 0)
    return b + np.random.default_rng(K + pool).integers(0, 256, size=K * stride, dtype=np.uint8).tobytes()


INNER = engine_v2(16, False, {}, (1, 1), {(0, 10): 0 | tg.HOT, (1, 10): 1 | tg.OWN})
GOOD_LIST = [(FAR, BASE, 1 | tg.OWN), (FAR + 1, BASE, 2 | tg.OWN), (BASE, FAR, 3 | tg.OWN)]


def graph_v2(glob_lists, refcount=(1, 1, 1, 1), pool=4 * DIM * DIM):
    glob = engine_v2(pool, True, glob_lists, refcount, {(0, 10): 0 | tg.OWN}, l2=0.05)
    return frame(MARKER + tg.graph_payload(inner=INNER, glob=glob), kind=tg.KIND, version=2)


def test_kind4_file_with_a_parked_grown_global_map_is_read(api, tmp_path):
    p = tmp_path / "ok.ckpt"
    p.write_bytes(graph_v2({0: GOOD_LIST}))       # pool 256 > dir_dim^2 = 64, three parked patches
    tg._expect_valid(api, p)


@pytest.mark.parametrize("name,lists,refcount,msg", [
    ("unsorted", {0: [GOOD_LIST[1], GOOD_LIST[0], GOOD_LIST[2]]}, (1, 1, 1, 1), "not strictly sorted"),
    ("duplicate", {0: [GOOD_LIST[0], GOOD_LIST[0]]}, (1, 2), "not strictly sorted"),
    ("inside the window", {0: [(BASE + 1, BASE + 2, 1)]}, (1, 1), "inside the saved window"),
    ("slot past K", {0: [(FAR, BASE, 4)]}, (1, 1, 1, 1), "past the saved slots"),
    ("unknown flag", {0: [(FAR, BASE, 1 | (1 << 27))]}, (1, 1), "unknown flag bits"),
    ("reference count", {0: GOOD_LIST}, (1, 1, 1, 2), "reference count differs"),
])
def test_malformed_parked_lists_of_the_global_map_are_refused(api, tmp_path, name, lists, refcount, msg):
    p = tmp_path / "bad.ckpt"
    p.write_bytes(graph_v2(lists, refcount=refcount))
    tg._expect_bad(api, p, msg=msg)


def test_global_map_pool_must_hold_its_slots_and_stay_below_the_slot_cap(api, tmp_path):
    p = tmp_path / "bad.ckpt"
    p.write_bytes(graph_v2({0: GOOD_LIST}, pool=3))
    tg._expect_bad(api, p, msg="more used slots than pool slots")
    p.write_bytes(graph_v2({0: GOOD_LIST}, pool=(1 << 24) - 1))
    tg._expect_bad(api, p, msg="bad pool size")


# ---- C-ABI ------------------------------------------------------------------------------------------------------------------------
NEW = ["lama_om_set_follow", "lama_om_get_window", "lama_om_get_pool"]


def test_new_entry_points_are_declared_and_exported(api):
    src = open(os.path.join(ROOT, "include", "lama_b200.h")).read()
    L = api.lib()
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, src) and n in api.EXPORTED_SYMBOLS and hasattr(L, n), n


def test_new_entry_points_refuse_null_arguments(api):
    L = api.lib()
    null = C.c_void_p(None)
    b2 = (C.c_int32 * 2)()
    d = C.c_int32(0)
    c3 = (C.c_uint64 * 3)()
    for fn, args in [(L.lama_om_set_follow, (null, C.c_int(1))), (L.lama_om_get_window, (null, b2, C.byref(d), c3)),
                     (L.lama_om_get_pool, (null, c3))]:
        fn.restype = C.c_int
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0


def test_following_map_needs_a_gpu_or_fails_loudly(api):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.LamaError) as e:
        api.FrequencyOccupancyMap(0.05, follow=True)
    assert e.value.code == -3


def test_shim_declares_the_map_window_and_pool(tmp_path):
    src = tmp_path / "shim.cpp"
    src.write_text('#include "lama_b200_shim.hpp"\nint main() { lama_om* m = nullptr; if (m) { lama_b200_shim::occupancyMapSetFollow(m, true);'
                   ' auto w = lama_b200_shim::occupancyMapWindow(m); uint64_t p[2]; lama_b200_shim::occupancyMapPool(m, p); return (int)w.dim; }'
                   ' return 0; }\n')
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])
