"""CPU tests of the moving window of the 2-D maps: window_shift_core.h (the per-entry logic of k_shift_count / k_shift_apply) and
window_guard.h (where PFSlam2D / Slam2D put the window before an update), through a host build of the same headers
(tests/emu/window_shift_emu.cpp), against a plain Python model."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HOT, OWN = 1 << 28, 1 << 29
OFF = 1321122 * 32   # kMapOffsetCells


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("window_shift_emu") / "libwindow_shift_emu.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so,
                           os.path.join(HERE, "emu", "window_shift_emu.cpp")])
    L = C.CDLL(so)
    L.emu_shift.restype = C.c_int
    L.emu_park_find.restype = C.c_int32
    L.emu_window_guard.restype = C.c_int
    L.emu_guard_box.restype = None
    L.emu_shift_scratch_check.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _shift(L, base, dim, nbase, dirs, parked):
    d = dirs.copy()
    pk = np.ascontiguousarray(parked, np.int32).reshape(-1, 3)
    out = np.zeros((len(pk) + dim * dim, 3), np.int32)
    ent = C.c_int(0)
    n = L.emu_shift(base[0], base[1], dim, nbase[0], nbase[1], _p(d), _p(pk), len(pk), _p(out), C.byref(ent))
    return d, out[:n].copy(), ent.value


def _all_entries(base, dim, dirs, parked):
    m = {}
    for i, e in enumerate(dirs):
        if e >= 0:
            m[(base[0] + i % dim, base[1] + i // dim)] = int(e)
    for px, py, e in parked:
        assert (px, py) not in m
        m[(int(px), int(py))] = int(e)
    return m


def _model(nbase, dim, entries):
    d = np.full(dim * dim, -1, np.int32)
    rest = []
    for (px, py), e in entries.items():
        x, y = px - nbase[0], py - nbase[1]
        if 0 <= x < dim and 0 <= y < dim:
            d[y * dim + x] = e
        else:
            rest.append((py, px, e))
    rest.sort()
    return d, np.array([(px, py, e) for py, px, e in rest], np.int32).reshape(-1, 3)


def _random_map(rng, base, dim, n_far):
    dirs = np.where(rng.random(dim * dim) < 0.4, rng.integers(0, 1 << 20, dim * dim), -1).astype(np.int32)
    flags = rng.integers(0, 4, dim * dim)
    dirs = np.where(dirs >= 0, dirs | np.where(flags & 1, HOT, 0) | np.where(flags & 2, OWN, 0), -1).astype(np.int32)
    far = set()
    while len(far) < n_far:
        px, py = (int(v) for v in rng.integers(-3 * dim, 4 * dim, 2))
        if not (0 <= px < dim and 0 <= py < dim):
            far.add((base[0] + px, base[1] + py))
    parked = sorted(((py, px) for px, py in far))
    parked = np.array([(px, py, int(rng.integers(0, 1 << 20)) | OWN) for py, px in parked], np.int32).reshape(-1, 3)
    return dirs, parked


@pytest.mark.parametrize("dim", [8, 16, 32])
def test_shift_matches_the_model_and_its_inverse_restores(emu, dim):
    rng = np.random.default_rng(dim)
    for trial in range(60):
        base = (5000 + int(rng.integers(0, 50)), 7000 + int(rng.integers(0, 50)))
        dirs, parked = _random_map(rng, base, dim, int(rng.integers(0, 200)))
        before = _all_entries(base, dim, dirs, parked)
        step = rng.integers(-2 * dim, 2 * dim + 1, 2) if trial % 3 else rng.integers(-2, 3, 2)
        nbase = (base[0] + int(step[0]), base[1] + int(step[1]))
        d, pk, entered = _shift(emu, base, dim, nbase, dirs, parked)
        md, mp = _model(nbase, dim, before)
        assert (d == md).all()
        assert (pk == mp).all()
        # entries conserved with their flags, no parked entry inside the window, the list sorted by (y, x)
        assert _all_entries(nbase, dim, d, pk) == before
        for px, py, _ in pk:
            assert not (0 <= px - nbase[0] < dim and 0 <= py - nbase[1] < dim)
        keys = [(int(py), int(px)) for px, py, _ in pk]
        assert keys == sorted(set(keys))
        assert entered == sum(1 for px, py, _ in parked if 0 <= px - nbase[0] < dim and 0 <= py - nbase[1] < dim)
        # the inverse shift gives back the directory and the list
        d2, pk2, _ = _shift(emu, nbase, dim, base, d, pk)
        assert (d2 == dirs).all() and (pk2 == parked).all()


def test_park_find_resolves_every_parked_patch(emu):
    rng = np.random.default_rng(3)
    _, parked = _random_map(rng, (100, 100), 16, 300)
    pk = np.ascontiguousarray(parked)
    for px, py, e in pk:
        assert emu.emu_park_find(_p(pk), len(pk), int(px), int(py)) == e
        assert emu.emu_park_find(_p(pk), len(pk), int(px) + 10000, int(py)) == -1
    assert emu.emu_park_find(_p(pk), 0, 100, 100) == -1


def _guard(L, base, dim, mn, mx, robot, res=0.05):
    mn, mx, robot = (np.array(v, float) for v in (mn, mx, robot))
    out = np.zeros(2, np.int32)
    d = L.emu_window_guard(base[0], base[1], dim, _p(mn), _p(mx), _p(robot), C.c_double(1.0 / res), _p(out))
    return d, (int(out[0]), int(out[1]))


def test_guard_decisions(emu):
    dim = 16                                   # 25.6 m at 0.05 m
    c = OFF // 32                              # the patch holding world 0
    base = (c - dim // 2, c - dim // 2)        # a window centred on the origin: patches [c - 8, c + 8)
    # inside: a 10 m box around the robot at the origin
    assert _guard(emu, base, dim, (-5, -5), (5, 5), (0, 0))[0] == 0
    # the robot drove to x = 15 m and its box leaves the window: the window is centred on the robot's patch
    d, nb = _guard(emu, base, dim, (10, -5), (20, 5), (15, 0))
    assert d == 1 and nb == ((OFF + 300) // 32 - dim // 2, base[1])
    # a box wider than the window fits no window: no shift
    assert _guard(emu, base, dim, (-13, -1), (13, 1), (0, 0))[0] == 2
    # a box that would fit a window, but not the one centred on the robot: no shift either (a beam past the window stays an error)
    assert _guard(emu, base, dim, (-1, -1), (12.85, 1), (0, 0))[0] == 2
    # the largest box the window centred on the robot holds, and one cell more
    d, nb = _guard(emu, base, dim, (102.4 - 12.8, 0.0), (102.4 + 12.8 - 0.01, 1.0), (102.4, 0.5))
    assert d == 1 and nb[0] == (OFF + 2048) // 32 - dim // 2
    assert _guard(emu, base, dim, (102.4 - 12.8 - 0.05, 0.0), (102.4 + 12.8 - 0.01, 1.0), (102.4, 0.5))[0] == 2


def test_guard_box_grows_by_spread_reach_and_slack(emu):
    pts = np.array([[4.0, 0.0, 0.0], [0.0, -3.0, 0.0]], float)
    one = np.array([1.0, 2.0, 0.0])
    mn, mx = np.zeros(2), np.zeros(2)
    emu.emu_guard_box(_p(one), 1, _p(pts), 2, C.c_double(0.05), C.c_uint32(10), _p(mn), _p(mx))
    g = (10 + 1 + 32) * 0.05
    assert np.allclose(mn, [1.0 - g, -1.0 - g]) and np.allclose(mx, [5.0 + g, 2.0 + g])
    # two particles 0.3 m apart with 0.1 rad between their headings: + 0.3 + 0.1 * range (4 m from the first pose)
    two = np.array([1.0, 2.0, 0.0, 1.3, 2.0, 0.1])
    emu.emu_guard_box(_p(two), 2, _p(pts), 2, C.c_double(0.05), C.c_uint32(10), _p(mn), _p(mx))
    g2 = g + 0.3 + 0.1 * 4.0
    assert np.allclose(mn, [1.0 - g2, -1.0 - g2]) and np.allclose(mx, [5.0 + g2, 2.0 + g2])


def test_shift_scratch_holds_lists_with_gaps(emu):
    """a prune shortens lists in place: list 0 kept 3 of its 10 entries, list 1 still starts at offset 10.  The enter-prefix scratch
    of a later shift must reach past the sum of the lengths (3 + 5 + 2 = 10) to the end of the furthest list"""
    for ol in ([(0, 3), (10, 5), (15, 0), (15, 2)], [(0, 0), (40, 1)], [(0, 7), (7, 7)], [(5, 0)]):
        a = np.array(ol, np.int32).reshape(-1)
        assert emu.emu_shift_scratch_check(_p(a), len(ol)) == 0, ol
    a = np.array([(0, 3), (10, 5), (15, 0), (15, 2)], np.int32)
    assert sum(l for _, l in a) + len(a) < max(o + l for o, l in a) + len(a)   # sizing by the lengths alone would be too short
