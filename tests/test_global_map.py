"""GraphSlam2D's global maps: generateOccupancyMap (src/graph_slam2d.cpp:131-164) with FrequencyOccupancyMap::prune
(src/sdm/frequency_occupancy_map.cpp:149-158), and generateCoarseDistanceMap (:166-186).
CPU: the oracle (tests/global_map_oracle.py) against hand cases and the oracle Slam2D, the call-sequence rules of the graph oracle, the
C-ABI boundary.  GPU: the device map (k_render_scans, lama_om_*) and the device GraphSlam2D's generators against the oracle."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import global_map_oracle as gmo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
O = gmo.OFFSET
ID = np.array([1.0, 0.0, 0.0, 0.0])


def _state(x, y, r):
    return np.array([math.cos(r), math.sin(r), x, y])


def _cells(m, mn, mx):
    return m.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1]))


# ---- CPU: the oracle -------------------------------------------------------------------------------------------------------------
def test_oracle_prune_rule_on_hand_cases():
    """visited == 1 and occupied in {0, 1} -> {0, 0}, known bit kept; anything else stays; a cell can be pruned again in a later call"""
    m = gmo.OccupancyMap(1.0)
    # cell (1, 0): one hit; (2, 0): one miss (on the ray to (3, 0)); (3, 0): hit twice; (5, 0) with hit + miss
    scans = [np.array([[1.0, 0, 0]]), np.array([[3.0, 0, 0]]), np.array([[3.0, 0, 0]])]
    m.insert_scans(scans[:1], [ID], full=False)
    m.insert_scans(scans[1:], [ID, ID], full=True)
    base = O
    e = m.export(base, base, 4, 1)
    assert e["visited"][0].tolist() == [0, 3, 2, 2] and e["occupied"][0].tolist() == [0, 1, 0, 2]
    m2 = gmo.OccupancyMap(1.0)
    m2.insert_scans(scans[:1], [ID], full=False)        # one hit on (1, 0)
    m2.prune()
    e = m2.export(base, base, 4, 1)
    assert e["visited"][0, 1] == 0 and e["occupied"][0, 1] == 0 and e["known"][0, 1] == 1
    m2.insert_scans(scans[:1], [ID], full=False)        # hit again after the prune: visited 1, occupied 1 -> pruned twice
    m2.prune()
    e = m2.export(base, base, 4, 1)
    assert (e["visited"][0, 1], e["occupied"][0, 1], e["known"][0, 1]) == (0, 0, 1)
    m2.insert_scans(scans[1:2], [ID], full=True)        # (1, 0) and (2, 0) one miss each, (3, 0) one hit
    m2.insert_scans(scans[1:2], [ID], full=True)        # once more before the prune: visited 2 everywhere -> kept
    m2.prune()
    e = m2.export(base, base, 4, 1)
    assert e["visited"][0].tolist() == [0, 2, 2, 2] and e["occupied"][0].tolist() == [0, 0, 0, 2]
    p, f = m2.query(np.array([[base + 1, base], [base + 3, base], [base + 9, base]], np.uint32))
    assert f.tolist() == [1, 2, 4] and p[2] == 0.25


def test_oracle_render_of_one_scan_is_slam2d_first_scan_before_prune(po, synth):
    """one scan cast with `full` at Slam2D's resolution = the oracle Slam2D's first-scan occupancy counters"""
    ds = synth.make_dataset("room", 1, n_beams=360)
    s = po.Slam2D(po.SlamOptions.defaults())
    s.set_pose(*ds.truth[0])
    assert s.update(ds.scans[0], ds.odom[0])
    m = gmo.OccupancyMap(0.05)
    m.insert_scans([ds.scans[0]], [po.se2_from_xyr(*ds.truth[0])], full=True)
    n, mn, mx = s.occ_bounds()
    nm, mn2, mx2 = m.bounds()
    assert n == nm and (mn == mn2).all() and (mx == mx2).all()
    a, b = s.export_occ(mn[0], mn[1], int(mx[0] - mn[0]), int(mx[1] - mn[1])), _cells(m, mn, mx)
    for k in ("occupied", "visited", "known"):
        assert (a[k] == b[k]).all(), k


def test_graph_oracle_call_sequence_rules(po, synth):
    """resolution fixed at creation, all keys cast again after every optimisation, a call without new keys only prunes"""
    ds = synth.make_dataset("loop", 1600, n_beams=360)
    g = gmo.GraphSlam2D()
    g.Init(*ds.truth[0])
    for t in range(60):
        g.update(ds.scans[t], ds.odom[t], float(t))
    m1 = g.generateOccupancyMap(full=False)
    assert m1.resolution == 0.1 and g.mapping_keyid == len(g.keys)
    before = _cells(m1, *m1.bounds()[1:])
    m2 = g.generateOccupancyMap(full=True)                 # no new keys: the same map, only pruned again
    assert m2 is m1 and m2.resolution == 0.1
    after = _cells(m2, *m2.bounds()[1:])
    assert all((before[k] == after[k]).all() for k in before)
    n_opt = len(g.optimizations)
    for t in range(60, ds.n_scans):
        g.update(ds.scans[t], ds.odom[t], float(t))
        if len(g.optimizations) > n_opt:
            break
    assert len(g.optimizations) > n_opt and g.mapping_keyid == 0   # optimizePoseGraph reset it
    m3 = g.generateOccupancyMap(full=True)
    assert m3 is not m1 and m3.resolution == 0.05
    ref = gmo.OccupancyMap(0.05)                               # every key cast again at its corrected pose
    ref.insert_scans([k["pts"] for k in g.keys], [k["pose"] for k in g.keys], True)
    ref.prune()
    assert ref.patches() == m3.patches()
    a, b = _cells(ref, *ref.bounds()[1:]), _cells(m3, *m3.bounds()[1:])
    assert all((a[k] == b[k]).all() for k in a)


def test_coarse_obstacle_order_is_directory_then_cell_order():
    occ = dict(occupied=np.zeros((64, 64), np.uint16), visited=np.zeros((64, 64), np.uint16), known=np.zeros((64, 64), np.uint8))
    for (x, y) in ((40, 3), (2, 5), (1, 40), (33, 33)):
        occ["occupied"][y, x] = occ["visited"][y, x] = occ["known"][y, x] = 1
    cells = gmo.coarse_obstacles(occ, occ["known"], np.array([O, O], np.uint32), 0.05)
    assert [(int(c[0]) - O, int(c[1]) - O) for c in cells] == [(1, 3), (20, 2), (1, 20), (17, 17)]   # patch (0,0), (1,0), (0,1), (1,1)


# ---- CPU: C-ABI -------------------------------------------------------------------------------------------------------------------
def test_header_declares_the_global_map_entry_points(api):
    src = open(os.path.join(ROOT, "include", "lama_b200.h")).read()
    assert "typedef struct lama_om lama_om;" in src
    names = ["lama_om_create", "lama_om_destroy", "lama_om_insert_scans", "lama_om_prune", "lama_om_resolution", "lama_om_bounds", "lama_om_query",
             "lama_om_export", "lama_om_write", "lama_om_export_image", "lama_om_kernel_times", "lama_graph_generate_occupancy_map",
             "lama_graph_generate_coarse_distance_map"]
    L = api.lib()
    for n in names:
        assert re.search(r"\b%s\s*\(" % n, src) and n in api.EXPORTED_SYMBOLS and hasattr(L, n), n


def test_global_map_entry_points_refuse_null_arguments(api):
    L = api.lib()
    null = C.c_void_p(None)
    n = C.c_int(0)
    u2 = (C.c_uint32 * 2)()
    d = C.c_double(0)
    calls = [
        (L.lama_om_create, (C.c_double(0.05), C.c_uint32(32), null, null, null)),
        (L.lama_om_insert_scans, (null, null, null, C.c_int(0), null, null, null, C.c_int(1), null)),
        (L.lama_om_prune, (null,)),
        (L.lama_om_resolution, (null, C.byref(d))),
        (L.lama_om_bounds, (null, u2, u2, C.byref(n))),
        (L.lama_om_query, (null, null, C.c_int(0), null, null)),
        (L.lama_om_export, (null, C.c_uint32(0), C.c_uint32(0), C.c_int(1), C.c_int(1), null, null, null)),
        (L.lama_om_write, (null, C.c_char_p(b"x.sdm"))),
        (L.lama_om_export_image, (null, null, C.c_size_t(0), null)),
        (L.lama_om_kernel_times, (null, null, null)),
        (L.lama_graph_generate_occupancy_map, (null, C.c_int(1), null)),
        (L.lama_graph_generate_coarse_distance_map, (null, null, null)),
    ]
    for fn, args in calls:
        fn.restype = C.c_int
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0
    assert L.lama_om_destroy(null) == 0


def test_occupancy_map_needs_a_gpu_or_fails_loudly(api):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.LamaError) as e:
        api.FrequencyOccupancyMap(0.05)
    assert e.value.code == -3                    # LAMA_ERR_NO_DEVICE


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------
def _same_map(g, o, tmp_path=None, query=True):
    ng, mn, mx = g.bounds()
    no, mn2, mx2 = o.bounds()
    assert ng == no and (mn == mn2).all() and (mx == mx2).all()
    if ng == 0:
        return
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g.export(int(mn[0]), int(mn[1]), w, h), o.export(int(mn[0]), int(mn[1]), w, h)
    for k in ("occupied", "visited", "known"):
        assert (a[k] == b[k]).all(), k
    assert gmo.patch_keys(mn, mx, a["known"].astype(bool) | (a["visited"] > 0)) <= o.patches()
    if query:
        ys, xs = np.mgrid[0:h:7, 0:w:5]
        cells = np.stack([xs.ravel() + mn[0], ys.ravel() + mn[1]], 1).astype(np.uint32)
        pg, fg = g.query(cells)
        po_, fo = o.query(cells)
        assert (fg == fo).all() and (pg == po_).all()
    if tmp_path is not None:
        from test_sdm_io import _same_files
        a_, b_ = tmp_path / "g.sdm", tmp_path / "o.sdm"
        g.write(a_)
        assert o.write(b_)
        f = _same_files(a_, b_)
        assert set(f["patches"]) == o.patches()        # exactly the patches that hold a touched cell
        assert (g.exportImage() == o.image()).all()


def _posed_scans(synth, n, beams, seed, spread=4.0):
    rng = np.random.default_rng(seed)
    ds = synth.make_dataset("room", 2, n_beams=beams)
    scans, states = [], []
    for k in range(n):
        x, y, r = rng.uniform(-spread, spread), rng.uniform(-spread, spread), rng.uniform(-math.pi, math.pi)
        scans.append(ds.scans[k % 2] * rng.uniform(0.3, 1.0))
        states.append(_state(x, y, r))
    return scans, np.array(states)


@pytest.mark.gpu
def test_device_insert_scans_equals_oracle(gpu_api, synth, tmp_path):
    """posed scans around negative and positive coordinates, across patch boundaries, a tilted sensor, full on and off, several
    insert + prune rounds: every cell, bounds, patch set, query flags, .sdm file and image"""
    for res in (0.05, 0.1):
        g = gpu_api.FrequencyOccupancyMap(res, center=(-1.0, 0.5))
        o = gmo.OccupancyMap(res)
        assert g.resolution == res
        for rnd in range(4):
            scans, states = _posed_scans(synth, 12, 361, seed=10 * rnd + int(res * 100))
            origins = np.tile([0.1, -0.05, 0.3], (len(scans), 1))
            quats = np.tile([0.0, 0.0, 0.0, 1.0], (len(scans), 1))
            if rnd == 2:   # tilted sensor: beams leave their z plane and take the 3-axis walk
                quats[::2] = [math.sin(0.05), 0.0, 0.0, math.cos(0.05)]
            full = rnd != 1
            cg = g.insertScans(scans, states, full=full, origins=origins, quats=quats)
            co = o.insert_scans(scans, states, full, origins=origins, quats=quats)
            assert cg == co
            _same_map(g, o)
            g.prune(); o.prune()
            _same_map(g, o, tmp_path if rnd == 3 else None)


@pytest.mark.gpu
def test_device_large_render_equals_oracle(gpu_api, synth):
    scans, states = _posed_scans(synth, 2000, 1080, seed=3, spread=12.0)
    g = gpu_api.FrequencyOccupancyMap(0.05)
    o = gmo.OccupancyMap(0.05)
    assert g.insertScans(scans, states, full=True) == o.insert_scans(scans, states, True)
    _same_map(g, o, query=False)


@pytest.mark.gpu
def test_device_window_overflow_is_an_error_not_an_access(gpu_api, synth):
    g = gpu_api.FrequencyOccupancyMap(0.05, dir_dim=8)   # 12.8 m window
    scans, states = _posed_scans(synth, 4, 360, seed=1, spread=30.0)
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertScans(scans, states, full=True)
    assert e.value.code == -4                  # LAMA_ERR_WINDOW from the status word


@pytest.mark.gpu
def test_device_graph_slam_global_maps_equal_oracle(gpu_api, po, synth, tmp_path):
    """two laps of the 30 m room: generateOccupancyMap every 100 scans with `full` alternating; after every call the whole map equals
    the oracle's render of the device's key poses under the same call sequence; generateCoarseDistanceMap equals the oracle's"""
    ds = synth.make_dataset("loop", 1600, n_beams=1080)
    g = gpu_api.GraphSlam2D()
    g.Init(*ds.truth[0])
    ref = None
    keyid = 0
    opts_seen = 0
    handle = None
    calls = 0
    for t in range(ds.n_scans):
        g.update(ds.scans[t], ds.odom[t], float(t))
        if t % 100 != 99:
            continue
        full = (calls % 2) == 0
        calls += 1
        st = g.stats()
        if st["optimizations"] > opts_seen:          # mapping_keyid = 0 after every optimisation (:428)
            opts_seen = st["optimizations"]
            keyid = 0
        m = g.generateOccupancyMap(full=full)
        if handle is None:
            handle = m
        cor, _, _ = g.keyPoses()
        if keyid == 0:
            ref = gmo.OccupancyMap(0.05 if full else 0.1)
        assert m.resolution == ref.resolution and handle.resolution == ref.resolution   # the first handle follows the recreated map
        new = range(keyid, len(cor))
        ref.insert_scans([g.keyCloud(i)[0] for i in new], [_state(*cor[i]) for i in new], full, thetas=cor[list(new), 2] if len(new) else None)
        ref.prune()
        keyid = len(cor)
        _same_map(m, ref, tmp_path if calls == 4 else None, query=calls == 4)
    assert opts_seen >= 1
    # the coarse distance map of the inner Slam2D's current local map
    slam = g.slam
    n1, a0, a1 = slam.mapBounds(1)
    n0, b0, b1 = slam.mapBounds(0)
    mn, mx = np.minimum(a0, b0), np.maximum(a1, b1)
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    cells = gmo.coarse_obstacles(slam.exportOccupancy(int(mn[0]), int(mn[1]), w, h), slam.exportDistance(int(mn[0]), int(mn[1]), w, h)["known"], mn, 0.05)
    od = po.DDM(0.1, 32, 5.0)
    od.add(cells)
    processed = od.update()
    dm = g.generateCoarseDistanceMap()
    assert len(cells) > 100 and dm.processed == processed and dm.max_sqdist == 2500
    n, mn, mx = od.bounds()
    ng, mng, mxg = dm.bounds()
    assert n == ng and (mn == mng).all() and (mx == mxg).all()
    a, b = dm.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1])), od.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1]))
    for k in ("sqdist", "valid", "ox", "oy", "known"):
        assert (a[k] == b[k]).all(), k
