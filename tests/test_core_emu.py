"""CPU tests of the product's core logic (lama_core.h / ddm_core.h / ray_core.h / match_core.h) through the
test-only host emulation in tests/emu: same headers as the CUDA kernels, compared with the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
O = 1321122 * 32


@pytest.fixture(scope="module")
def emu():
    subprocess.check_call(["make", "-C", os.path.join(HERE, "emu"), "-s"])
    L = C.CDLL(os.path.join(HERE, "emu", "_build", "liblama_emu.so"))
    L.emu_create.restype = C.c_void_p
    L.emu_create.argtypes = [C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_uint32, C.c_int]
    L.emu_dm_apply.restype = C.c_uint32
    L.emu_prob_replay.restype = C.c_float
    L.emu_freq_replay.restype = C.c_uint32
    for f in ("emu_destroy", "emu_set_pose", "emu_get_state", "emu_counters", "emu_slam_update", "emu_export_dm", "emu_export_occ", "emu_dm_apply", "emu_set_pull",
              "emu_pull_fallbacks", "emu_freq_replay"):
        getattr(L, f).argtypes = None
    return L


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _export_dm(L, h, x0, y0, w, hh):
    o = dict(sqdist=np.zeros((hh, w), np.uint16), valid=np.zeros((hh, w), np.uint8), known=np.zeros((hh, w), np.uint8),
             ox=np.zeros((hh, w), np.int16), oy=np.zeros((hh, w), np.int16), queued=np.zeros((hh, w), np.uint8))
    L.emu_export_dm(C.c_void_p(h), C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(hh), _vp(o["sqdist"]), _vp(o["valid"]), _vp(o["known"]),
                    _vp(o["ox"]), _vp(o["oy"]), _vp(o["queued"]))
    return o


def _export_occ(L, h, x0, y0, w, hh):
    o = dict(occupied=np.zeros((hh, w), np.uint16), visited=np.zeros((hh, w), np.uint16), obstacle=np.zeros((hh, w), np.uint8))
    L.emu_export_occ(C.c_void_p(h), C.c_uint32(x0), C.c_uint32(y0), C.c_int(w), C.c_int(hh), _vp(o["occupied"]), _vp(o["visited"]), _vp(o["obstacle"]))
    return o


def test_heap_is_bit_faithful_to_std_priority_queue(emu):
    # many ties (small priority range) are what makes the pop order implementation defined
    for seed, n, rng in ((1, 20000, 4), (2, 20000, 1), (3, 50000, 100), (4, 3000, 2), (5, 100000, 401)):
        assert emu.emu_heap_check(C.c_uint32(seed), C.c_int(n), C.c_int(rng)) == 0


def test_kernel_segment_walk_equals_iterative_bresenham(emu):
    """ray_core.h SegWalk (what k_raycast's lanes execute: packed cell, major/minor state, closed-form start of a 64-step segment)
    against Map::computeRay's iterative walk (map.cpp:198-227)"""
    assert emu.emu_segwalk_check(C.c_int(150), C.c_uint32(0), C.c_int(0), C.c_int(0), C.c_int(64)) == 0      # all 301^2 beams incl. n = 0, 1, diagonals
    assert emu.emu_segwalk_check(C.c_int(40), C.c_uint32(0), C.c_int(0), C.c_int(0), C.c_int(7)) == 0        # odd segment length: every start offset
    assert emu.emu_segwalk_check(C.c_int(0), C.c_uint32(3), C.c_int(20000), C.c_int(2048), C.c_int(64)) == 0  # dir_dim 64 windows
    assert emu.emu_segwalk_check(C.c_int(0), C.c_uint32(4), C.c_int(20000), C.c_int(4096), C.c_int(64)) == 0  # the largest window (dir_dim 128)


def test_pull_raycast_counts_equal_iterative_bresenham(emu):
    """ray_pull.h (what k_ray_setup / k_ray_pull execute): class lists sorted by exact slope, patch marking, per-cell crossing counts (one beam range per class and patch, k(a) by exact reciprocal division)
    and the per-cell runs with their step indices, against Map::computeRay's iterative walk (map.cpp:198-227) for every cell of the window"""
    emu.emu_pull_check.restype = C.c_int
    assert emu.emu_magic_check(C.c_int(4096)) == 0   # the exact reciprocal division behind k(a) = floor((2 a d + n) / (2 n))
    for mode in range(4):   # scan-like fans, random end cells, very short beams (n = 0, 1, 2), axes and diagonals
        for seed, n, dim in ((1, 1080, 16), (2, 360, 8), (3, 2000, 32), (4, 50, 8), (5, 1080, 64), (6, 720, 128)):
            assert emu.emu_pull_check(C.c_uint32(seed * 7 + mode), C.c_int(n), C.c_int(mode), C.c_int(dim)) == 0, (mode, seed)


def test_packed_cell_addressing(emu):
    """k_raycast's packed-cell shortcuts (directory index, byte offset in the patch, log key) == dir_index / cell_index / cell_key"""
    for log2dim in (3, 6, 7):
        assert emu.emu_packed_cell_check(C.c_int(log2dim)) == 0


def test_register_only_ldlt_equals_the_indexed_formulation(emu):
    """match_core.h ldlt_solve3 (what k_match runs: no run-time indices, so no local memory on the device) == ldlt_solve3_indexed, bit for bit"""
    assert emu.emu_ldlt_check(C.c_uint32(3), C.c_int(400000)) == 0


def test_se2_host_math_equals_oracle_bitwise(emu, po):
    rng = np.random.default_rng(0)
    out = np.zeros(4)
    for _ in range(200):
        a = po.se2_from_xyr(*rng.uniform(-3, 3, 3))
        b = po.se2_from_xyr(*rng.uniform(-3, 3, 3))
        emu.emu_se2(C.c_int(0), _vp(a), _vp(b), _vp(out))
        assert (out == po.se2_mul(a, b)).all()
        emu.emu_se2(C.c_int(1), _vp(a), None, _vp(out))
        assert (out == po.se2_inv(a)).all()
        h = np.ascontiguousarray(rng.uniform(-0.2, 0.2, 3))
        emu.emu_se2(C.c_int(2), _vp(h), None, _vp(out))
        assert (out == po.se2_exp(h)).all()


@pytest.mark.parametrize("l2", [0.5, 1.0])
def test_brushfire_core_equals_oracle_on_add_remove_stress(emu, po, l2):
    h = emu.emu_create(0.05, l2, 3.2, 3.2, 16, 0.5, 0.5, 100, 0)
    o = po.DDM(l2_max=l2)
    rng = np.random.default_rng(7)
    W = 128
    occ = np.zeros((W, W), bool)
    for it in range(60):
        mode = rng.integers(0, 3)
        n = int(rng.integers(1, 50))
        if mode == 0:
            pts = rng.integers(24, W - 24, size=(n, 2))
        elif mode == 1:
            x0, y0 = rng.integers(24, W - 24, 2); dx, dy = rng.integers(-1, 2, 2)
            pts = np.array([(x0 + k * dx, y0 + k * dy) for k in range(n)]); pts = pts[(pts.min(1) >= 24) & (pts.max(1) < W - 24)]
        else:
            pts = np.argwhere(occ)[:, ::-1]
            if len(pts):
                pts = pts[rng.choice(len(pts), size=min(len(pts), n), replace=False)]
        if len(pts) == 0:
            continue
        cells = np.ascontiguousarray((pts + O).astype(np.uint32))
        kinds = np.full(len(cells), 0 if mode == 2 else 1, np.uint8)
        if mode == 2:
            o.remove(cells); occ[pts[:, 1], pts[:, 0]] = False
        else:
            o.add(cells); occ[pts[:, 1], pts[:, 0]] = True
        pops_e = emu.emu_dm_apply(C.c_void_p(h), _vp(cells), _vp(kinds), C.c_int(len(cells)))
        assert pops_e == o.update()
        a, b = _export_dm(emu, h, O, O, W, W), o.export(O, O, W, W)
        for k in ("sqdist", "valid", "ox", "oy", "queued"):
            assert (a[k] == b[k]).all(), (it, k)
    emu.emu_destroy(C.c_void_p(h))


@pytest.mark.parametrize("name,beams,T,shuffle", [("room", 360, 25, 0), ("room", 360, 25, 12345), ("corridor", 240, 20, 99), ("room", 360, 25, "pull"),
                                                  ("corridor", 240, 20, "pull"), ("loop", 1080, 12, "pull")])
def test_emulated_slam_equals_oracle(emu, po, synth, name, beams, T, shuffle):
    """Packed atomics in a SHUFFLED beam order + ordered replay + sequential brushfire == the reference's
    strictly sequential update (cells bit-exact), and the fused one-evaluation-per-iteration solver == Solver::solve."""
    ds = synth.make_dataset(name, T, n_beams=beams)
    t0 = ds.truth[0]
    h = emu.emu_create(0.05, 0.5, t0[0], t0[1], 64, 0.05, 0.05, 100, 0)
    emu.emu_set_pose(C.c_void_p(h), C.c_double(t0[0]), C.c_double(t0[1]), C.c_double(t0[2]))
    pull = shuffle == "pull"   # the pull form of the ray cast (ray_pull.h) instead of per-beam walks
    if pull:
        emu.emu_set_pull(C.c_void_p(h), C.c_int(1))
        shuffle = 0
    o = po.Slam2D(po.SlamOptions.defaults(trans_thresh=0.05, rot_thresh=0.05))
    o.set_pose(*t0)
    st = np.zeros(4)
    ctr = np.zeros(7, np.uint32)
    for t in range(T):
        pts = np.ascontiguousarray(ds.scans[t]); od = np.ascontiguousarray(ds.odom[t])
        a = emu.emu_slam_update(C.c_void_p(h), _vp(pts), C.c_int(beams), _vp(od), C.c_uint32(shuffle))
        b = o.update(ds.scans[t], ds.odom[t])
        assert bool(a) == b
        emu.emu_get_state(C.c_void_p(h), _vp(st))
        assert np.abs(st - o.state()).max() < 1e-12
        emu.emu_counters(C.c_void_p(h), _vp(ctr))
        last, _ = o.counters()
        assert ctr[6] == 0
        assert (int(ctr[0]), int(ctr[1]), int(ctr[2]), int(ctr[5])) == (last["evals"], last["ray_cells"], last["dm_pops"], last["gn_iters"])
    n, mn, mx = o.dm_bounds(); w, hh = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = _export_dm(emu, h, int(mn[0]), int(mn[1]), w, hh), o.export_dm(mn[0], mn[1], w, hh)
    for k in ("sqdist", "valid", "ox", "oy", "queued", "known"):
        assert (a[k] == b[k]).all(), k
    n, mn, mx = o.occ_bounds(); w, hh = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = _export_occ(emu, h, int(mn[0]), int(mn[1]), w, hh), o.export_occ(mn[0], mn[1], w, hh)
    assert (a["occupied"] == b["occupied"]).all() and (a["visited"] == b["visited"]).all()
    # the obstacle mirror bit of the occupancy word equals "distance cell is an obstacle"
    d = _export_dm(emu, h, int(mn[0]), int(mn[1]), w, hh)
    assert (a["obstacle"].astype(bool) == ((d["valid"] == 1) & (d["sqdist"] == 0))).all()
    if pull:
        emu.emu_pull_fallbacks.restype = C.c_uint32
        assert emu.emu_pull_fallbacks(C.c_void_p(h)) == 0   # every scan went through the pull path
    emu.emu_destroy(C.c_void_p(h))


def _frequency_cell(occ, vis, kinds, obstacle):
    """FrequencyOccupancyMap::setOccupied / setFree (frequency_occupancy_map.cpp:65-91) on two independent uint16 counters, and the
    no-op rules of addObstacle / removeObstacle (dynamic_distance_map.cpp:217-218,233-234): the final counters, the obstacle flag and
    the event of every touch (1 add, 2 remove, 0 none)"""
    ev = np.zeros(len(kinds), np.uint8)
    for i, k in enumerate(kinds):
        if k:
            was = vis != 0 and 4 * occ > vis
            occ, vis = (occ + 1) & 0xFFFF, (vis + 1) & 0xFFFF
            if not was and vis != 0 and 4 * occ > vis and not obstacle:
                obstacle, ev[i] = True, 1
        else:
            was = vis != 0 and 4 * occ < vis
            vis = (vis + 1) & 0xFFFF
            if not was and vis != 0 and 4 * occ < vis and obstacle:
                obstacle, ev[i] = False, 2
    return occ, vis, obstacle, ev


def test_frequency_replay_takes_back_the_carry_of_a_wrapped_occupied_count(emu):
    """replay_cell (ray_core.h) on packed words whose `occupied` half wraps in this scan: a packed hit carries into `visited`, the
    reference's separate uint16 does not.  The stored word, the pre-scan state the replay starts from (seen through its events) and
    the obstacle flag must follow the two independent counters; the plain packed sum must differ wherever occupied wrapped."""
    rng = np.random.default_rng(21)
    cases = [(0xFFFF, 0xFFFF, [1]), (0xFFFF, 0x0000, [1]), (0xFFFE, 0x0010, [1, 1, 1]), (0x0000, 0x0000, [1] * 65535),
             (0xFFF0, 0x4000, [0] * 60000 + [1] * 16), (0x3FFF, 0xFFFF, [0, 1]), (0xFFFF, 0xFFFF, [0] * 3)]
    for _ in range(300):
        occ, vis = int(rng.choice([0xFFFF, 0xFFFE, 0xFF80, 0xC000, 0x4000, 0, 7])), int(rng.integers(0, 0x10000))
        n = int(rng.integers(1, 600))
        cases.append((occ, vis, (rng.random(n) < rng.choice([0.05, 0.3, 0.6, 1.0])).astype(np.uint8).tolist()))
    wrapped = 0
    for occ, vis, kinds in cases:
        k = np.ascontiguousarray(kinds, np.uint8)
        hits = int(k.sum())
        assert hits < 0x10000                                    # a cell takes at most one hit per beam and scan
        for obstacle_in in (0, 1):
            ev = np.zeros(len(k), np.uint8)
            ob = C.c_int(0)
            word = emu.emu_freq_replay(_vp(k), C.c_int(len(k)), C.c_uint32((vis << 16) | occ), C.c_int(obstacle_in), _vp(ev), C.byref(ob))
            o2, v2, flag, want = _frequency_cell(occ, vis, kinds, bool(obstacle_in))
            assert word == (v2 << 16) | o2, (occ, vis, hits, len(k))
            assert (ev == want).all() and bool(ob.value) == flag
            packed = (((vis << 16) | occ) + hits * 0x10001 + (len(k) - hits) * 0x10000) & 0xFFFFFFFF
            if occ + hits >= 0x10000:
                wrapped += 1
                assert packed >> 16 == (v2 + 1) & 0xFFFF             # without the correction visited is one ahead
            else:
                assert packed == word
    assert wrapped >= 20


def test_logodds_replay_equals_probabilistic_occupancy_map(emu, po):
    """replay_cell_prob == ProbabilisticOccupancyMap::setFree/setOccupied call by call (float cell, clamps, thresholds)"""
    rng = np.random.default_rng(4)
    cst = po.prob_constants()
    constants = np.array([cst["miss"], cst["hit"], cst["clamp_min"], cst["clamp_max"], cst["occ_thresh"]])
    for trial in range(200):
        n = int(rng.integers(1, 60))
        kinds = (rng.random(n) < rng.choice([0.1, 0.3, 0.5, 0.9])).astype(np.uint8)
        prob, changed = po.prob_sequence(kinds)
        # distance-map side of the reference: addObstacle / removeObstacle are no-ops when the flag already matches
        flag, want = False, np.zeros(n, np.uint8)
        for i in range(n):
            if changed[i]:
                if kinds[i] and not flag:
                    flag, want[i] = True, 1
                elif not kinds[i] and flag:
                    flag, want[i] = False, 2
        ev = np.zeros(n, np.uint8)
        ob = C.c_int(0)
        p = emu.emu_prob_replay(_vp(kinds), C.c_int(n), _vp(constants), C.c_int(0), _vp(ev), C.byref(ob))
        assert np.float32(p) == prob[-1]
        assert (ev == want).all() and bool(ob.value) == flag
