"""The 2-D maps and the scan matcher across resolution and distance-map reach, up to the 63-cell limit of the packed distance cell.

The reach of a DynamicDistanceMap is ceil(l2_max * scale) cells (dynamic_distance_map.cpp:149-153).  The device packs a distance cell in
one word: 12-bit sqdist and 7-bit two's-complement obstacle offsets (lama_core.h), so 63 cells is the largest reach it accepts.  What
changes with reach and resolution: offsets near +-63, the max_sqdist + 1 entry distance table that k_match keeps in shared memory,
brushfire waves that cross two patch borders, the rounding of ceil(l2_max * scale), and the size of the brushfire heaps (k_brushfire
keeps their first entries in shared memory and moves a heap to global memory when it outgrows that part).

Every scenario has a CPU check that it does what its name says; the GPU tests compare the device with the oracle: every cell bit-exact,
update() return values, dm_pops and ray_cells per scan, poses within POSE_TOL."""
import ctypes as C
import math

import numpy as np
import pytest
from scipy import ndimage

from test_core_emu import _export_dm, _export_occ, _vp, emu  # noqa: F401  (emu: the host-emulation fixture)

O = 1321122 * 32
POSE_TOL = 1e-9
WALK, PULL = "0", "100000"   # LAMA_PULL_MAX_PARTICLES: the per-beam walk / the pull form of the ray cast for every particle count
SMEM_HEAP_CAP = 8192         # entries of the lower heap in shared memory (engine.cu)


def reach_of(res, l2):
    """DynamicDistanceMap::setMaxDistance: ceil(l2_max * scale) with scale = 1 / resolution, in double precision"""
    return math.ceil(l2 * (1.0 / res))


def l2_for(res, k):
    """the largest l2_max whose reach at `res` is k cells (k * res itself may round up to k + 1: 63 * 0.1 * 10 > 63)"""
    l2 = k * res
    while reach_of(res, l2) > k:
        l2 = float(np.nextafter(l2, 0.0))
    assert reach_of(res, l2) == k
    return l2


def cell(v, res):
    """Map::w2m of one world coordinate"""
    return int(np.uint32(v * (1.0 / res) + O + 0.5))


# ---- reach arithmetic -------------------------------------------------------------------------------------------------------------
RESOLUTIONS = (0.1, 0.05, 0.03, 0.025, 0.015)
REACHES = (1, 2, 31, 32, 33, 62, 63)


def reach_table():
    """(resolution, l2_max) for every wanted reach k at every resolution, with l2_max = k * resolution (whose product with the scale
    may or may not land on k exactly), plus pairs whose product lands just above a whole number (the reach rounds up)"""
    pairs = [(r, k * r) for r in RESOLUTIONS for k in REACHES]
    pairs += [(0.03, 0.93), (0.1, 0.7), (0.05, 0.15), (0.015, 0.93), (0.025, 0.775)]
    return pairs


def test_reach_table_covers_exact_and_rounded_up_products():
    pairs = reach_table()
    exact = [(r, l) for r, l in pairs if l * (1.0 / r) == math.floor(l * (1.0 / r))]
    above = [(r, l) for r, l in pairs if l * (1.0 / r) != math.floor(l * (1.0 / r))]
    assert {reach_of(r, l) for r, l in exact} >= set(REACHES)
    assert len(above) >= 5 and all(l * (1.0 / r) - math.floor(l * (1.0 / r)) < 1e-9 for r, l in above)   # just above a whole number
    assert 0.93 * (1.0 / 0.03) == 31.000000000000004 and reach_of(0.03, 0.93) == 32
    assert {r for r, _ in pairs} == set(RESOLUTIONS)


def test_reach_arithmetic_matches_the_oracle(po):
    for res, l2 in reach_table():
        k = reach_of(res, l2)
        if k > 63:
            continue
        assert po.DDM(res, l2_max=l2).max_sqdist == k * k, (res, l2)


# ---- the oracle at the largest reach ----------------------------------------------------------------------------------------------
def test_oracle_single_obstacle_at_reach_63_is_exact_edt(po):
    """one obstacle: the brushfire is exact, every valid cell is inside the 63-cell disc, offsets reach +-62 in both axes"""
    for res in (0.1, 0.025):
        d = po.DDM(res, l2_max=l2_for(res, 63))
        assert d.max_sqdist == 63 * 63
        c, W = 70, 141
        d.add(np.array([[O + c, O + c]], np.uint32))
        d.update()
        e = d.export(O, O, W, W)
        yy, xx = np.mgrid[0:W, 0:W]
        sq = (xx - c) ** 2 + (yy - c) ** 2
        want = sq < d.max_sqdist
        assert (e["valid"].astype(bool) == want).all()
        assert (e["sqdist"][want] == sq[want]).all()
        assert (e["ox"][want] == (c - xx)[want]).all() and (e["oy"][want] == (c - yy)[want]).all()
        for k in ("ox", "oy"):
            assert e[k][want].max() == 62 and e[k][want].min() == -62


def test_oracle_walls_at_reach_63_match_brute_force_edt(po):
    for res in (0.1, 0.025):
        W = 280   # 62 free cells on either side of each wall
        occ = np.zeros((W, W), bool)
        occ[80, 70:210] = True
        occ[80:200, 70] = True
        occ[160:166, 150:156] = True
        d = po.DDM(res, l2_max=l2_for(res, 63))
        d.add((np.argwhere(occ)[:, ::-1] + O).astype(np.uint32))
        assert d.update() > 0
        e = d.export(O, O, W, W)
        edt2 = np.rint(ndimage.distance_transform_edt(~occ) ** 2).astype(np.int64)
        want = edt2 < d.max_sqdist
        assert (e["valid"].astype(bool) == want).all()
        assert (e["sqdist"][want] == edt2[want]).all()
        assert e["ox"][want].max() == 62 and e["oy"][want].max() == 62 and e["ox"][want].min() == -62 and e["oy"][want].min() == -62


# ---- the heap-overflow scenario and the emulated Slam2D ------------------------------------------------------------------------------
# loop, 1 080 beams, 0.025 m, l2_max 1.5 (60 cells).  With dir_dim 64 the waves leave the 51 m window, and with max_beams 2 048 and
# dir_dim 128 the ray cast's shared memory exceeds 227 KB: both are reported errors, not what this scenario is about.
OVERFLOW = dict(name="loop", beams=1080, T=4, res=0.025, l2=1.5, dim=128)
EMU_CASES = [dict(name="room", beams=360, T=8, res=0.025, l2=1.5, dim=64), dict(name="room", beams=360, T=8, res=0.1, l2=6.0, dim=64),
             dict(name="room", beams=360, T=8, res=0.05, l2=3.15, dim=64), dict(name="room", beams=360, T=8, res=0.03, l2=0.93, dim=64),
             OVERFLOW]


def _emu_slam(emu, po, synth, name, beams, T, res, l2, dim):
    """the emulated Slam2D (the CUDA kernels' headers on the host) against the oracle, scan by scan and cell by cell; returns the
    largest lower / raise heap of any of its brushfires"""
    ds = synth.make_dataset(name, T, n_beams=beams)
    t0 = ds.truth[0]
    h = emu.emu_create(res, l2, t0[0], t0[1], dim, 0.05, 0.05, 100, 0)
    emu.emu_set_pose(C.c_void_p(h), C.c_double(t0[0]), C.c_double(t0[1]), C.c_double(t0[2]))
    o = po.Slam2D(po.SlamOptions.defaults(trans_thresh=0.05, rot_thresh=0.05, resolution=res, l2_max=l2))
    o.set_pose(*t0)
    st, ctr = np.zeros(4), np.zeros(7, np.uint32)
    for t in range(T):
        a = emu.emu_slam_update(C.c_void_p(h), _vp(np.ascontiguousarray(ds.scans[t])), C.c_int(beams), _vp(np.ascontiguousarray(ds.odom[t])), C.c_uint32(0))
        assert bool(a) == o.update(ds.scans[t], ds.odom[t]), t
        emu.emu_get_state(C.c_void_p(h), _vp(st))
        assert np.abs(st - o.state()).max() < 1e-12, t
        emu.emu_counters(C.c_void_p(h), _vp(ctr))
        last, _ = o.counters()
        assert ctr[6] == 0
        assert (int(ctr[0]), int(ctr[1]), int(ctr[2]), int(ctr[5])) == (last["evals"], last["ray_cells"], last["dm_pops"], last["gn_iters"]), t
    n, mn, mx = o.dm_bounds(); w, hh = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = _export_dm(emu, h, int(mn[0]), int(mn[1]), w, hh), o.export_dm(mn[0], mn[1], w, hh)
    for k in ("sqdist", "valid", "ox", "oy", "queued", "known"):
        assert (a[k] == b[k]).all(), k
    n, mn, mx = o.occ_bounds(); w, hh = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = _export_occ(emu, h, int(mn[0]), int(mn[1]), w, hh), o.export_occ(mn[0], mn[1], w, hh)
    assert (a["occupied"] == b["occupied"]).all() and (a["visited"] == b["visited"]).all()
    peak = np.zeros(2, np.uint32)
    emu.emu_heap_peak.argtypes = None
    emu.emu_heap_peak(C.c_void_p(h), _vp(peak))
    emu.emu_destroy(C.c_void_p(h))
    return int(peak[0]), int(peak[1])


@pytest.mark.parametrize("case", EMU_CASES, ids=lambda c: f"{c['name']}-{c['res']}-{c['l2']}")
def test_emulated_slam_equals_oracle_across_reach(emu, po, synth, case):
    peak = _emu_slam(emu, po, synth, **case)
    if case is OVERFLOW:
        assert peak[0] > SMEM_HEAP_CAP, peak   # the lower heap outgrows its shared-memory part: the scenario tests what its name says


# ---- GPU: DynamicDistanceMap add / remove stress ------------------------------------------------------------------------------------
DDM_TABLE = [(0.1, 6.3), (0.025, 1.575), (0.05, 3.15), (0.03, 0.93), (0.015, 0.945), (0.1, 0.1), (0.05, 1.65), (0.025, 0.05), (0.1, 3.1)]


def test_ddm_table_reaches():
    assert sorted({reach_of(r, l) for r, l in DDM_TABLE}) == [1, 2, 31, 32, 33, 63]
    assert {r for r, _ in DDM_TABLE} == set(RESOLUTIONS)


def _dm_equal(a, b, tag):
    for k in ("sqdist", "valid", "ox", "oy", "queued", "known"):
        assert (a[k] == b[k]).all(), (tag, k, int((a[k] != b[k]).sum()))


def ddm_stress_steps(reach, seed=11, n_steps=24):
    """(kind, cells) per update: random points, lines and removals over a 224-cell square that starts on a patch border, plus single
    obstacles next to patch borders whose waves (reach > 32) cross two borders; at most 2 048 cells per update"""
    rng = np.random.default_rng(seed)
    W, lo = 224, 32 * 2
    occ = np.zeros((W, W), bool)
    steps = []
    for it in range(n_steps):
        mode = it % 4 if it else 3
        n = int(rng.integers(1, 80))
        if mode == 0:
            pts = rng.integers(0, W, size=(n, 2))
        elif mode == 1:
            x0, y0 = rng.integers(0, W, 2); dx, dy = rng.integers(-1, 2, 2)
            pts = np.array([(x0 + k * dx, y0 + k * dy) for k in range(n)]); pts = pts[(pts.min(1) >= 0) & (pts.max(1) < W)]
        elif mode == 2:
            pts = np.argwhere(occ)[:, ::-1]
            if len(pts):
                pts = pts[rng.choice(len(pts), size=min(len(pts), n), replace=False)]
        else:   # next to the borders of the patches 1 and 2 away: a 33+ cell wave crosses two of them
            pts = np.array([(31, 31), (32, 95), (95, 32), (127, 128), (160, 191)])[: 1 + it % 5]
        if len(pts) == 0:
            continue
        occ[pts[:, 1], pts[:, 0]] = mode != 2
        steps.append((mode != 2, (pts + O + lo).astype(np.uint32)))
    return steps, W + 2 * lo, O


@pytest.mark.gpu
@pytest.mark.parametrize("res,l2", DDM_TABLE)
def test_ddm_add_remove_stress_across_reach(gpu_api, po, res, l2):
    g, o = gpu_api.DynamicDistanceMap(res, l2_max=l2), po.DDM(res, l2_max=l2)
    assert g.max_sqdist == o.max_sqdist == reach_of(res, l2) ** 2
    steps, W, x0 = ddm_stress_steps(reach_of(res, l2))
    for it, (add, cells) in enumerate(steps):
        assert len(cells) <= 2048
        if add:
            g.addObstacle(cells); o.add(cells)
        else:
            g.removeObstacle(cells); o.remove(cells)
        assert g.update() == o.update(), it
        _dm_equal(g.export(x0, x0, W, W), o.export(x0, x0, W, W), it)
    rng = np.random.default_rng(5)
    pts = np.zeros((3000, 3)); pts[:, :2] = rng.uniform(-0.3 * res, (W + 0.3) * res, size=(3000, 2))
    dg, gg = g.distance(pts); dc, gc = o.distance(pts)
    assert (dg == dc).all() and (gg == gc).all()


def test_ddm_stress_waves_cross_two_patch_borders(po):
    """CPU check of the stress scenario at reach 63: some obstacle's valid cells span three patches in x and in y"""
    res = 0.1
    o = po.DDM(res, l2_max=l2_for(res, 63))
    steps, W, x0 = ddm_stress_steps(63)
    add, cells = steps[0]
    o.add(cells); o.update()
    e = o.export(x0, x0, W, W)
    xs = np.nonzero(e["valid"].any(0))[0] + x0
    ys = np.nonzero(e["valid"].any(1))[0] + x0
    assert (xs.max() >> 5) - (cells[:, 0].min() >> 5) >= 2 or (cells[:, 0].max() >> 5) - (xs.min() >> 5) >= 2
    assert (ys.max() >> 5) - (cells[:, 1].min() >> 5) >= 2 or (cells[:, 1].max() >> 5) - (ys.min() >> 5) >= 2


# ---- GPU: the reach limit ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reach_63_is_accepted_and_64_refused_at_creation(gpu_api):
    for l2, ok in ((l2_for(0.05, 63), True), (l2_for(0.05, 64), False)):
        makers = [lambda: gpu_api.DynamicDistanceMap(0.05, l2_max=l2),
                  lambda: gpu_api.Slam2D(gpu_api.Slam2D.Options(l2_max=l2)),
                  lambda: gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(4, l2_max=l2, seed=1)),
                  lambda: gpu_api.Loc2D(gpu_api.Loc2D.Options(l2_max=l2))]
        for make in makers:
            if ok:
                make()
            else:
                with pytest.raises(gpu_api.LamaError) as e:
                    make()
                assert e.value.code == -1 and "63" in str(e.value)


# ---- GPU: the scan matcher at the edges of k_match ----------------------------------------------------------------------------------
BEAMS = (1, 31, 32, 33, 128, 129, 575, 576, 577, 1152, 1153, 4096)
MATCH_DEV = dict(dir_dim=32, max_beams=4096)   # a 4 096-beam scan fits the ray cast's shared memory with a 32-patch window


def match_block(n):
    """launch_match's block size: ceil(n / ceil(n / 576)) threads rounded up to a multiple of 32, at least 128"""
    rounds = -(-n // 576)
    return max(128, (-(-n // rounds) + 31) // 32 * 32)


def match_world(res):
    """obstacle cells of a room around the origin (walls 40 cells out, a pillar) and the sensor-frame points of a scan whose end cells
    fall (a) inside one patch, (b) on a cell with x & 31 == 31 or y & 31 == 31 (the bilinear stencil straddles a patch border), (c) in
    patches no obstacle wave reached (unallocated) and (d) outside the directory window"""
    walls = [(x, y) for x in range(-40, 41) for y in (-40, 40)] + [(x, y) for y in range(-40, 41) for x in (-40, 40)]
    walls += [(x, y) for x in range(10, 14) for y in range(-20, -16)]
    cells = np.array([(O + x, O + y) for x, y in walls], np.uint32)
    kinds = {}
    kinds["inside"] = [(O + x + f, O + y + g) for x, y in [(-38, 5), (20, 38), (-7, -37), (37, -12), (12, -15)] for f, g in ((0.2, 0.3), (0.5, 0.7))]
    kinds["straddle"] = [(O - 33 + 0.6, O + 10.4), (O + 31 + 0.5, O + 38.2), (O + 12.3, O - 33 + 0.8), (O + 38.5, O + 31 + 0.5), (O + 31.5, O - 33.5)]
    kinds["unallocated"] = [(O + 300.5, O + 200.5), (O - 400.2, O - 300.7), (O + 250.3, O - 450.1)]
    kinds["outside"] = [(O + 600.5, O + 3.5), (O - 3.5, O - 600.5), (O + 1000.5, O + 1000.5)]
    return cells, kinds


def match_scan(n, res, kinds):
    """n sensor-frame points (the sensor at the origin) cycling over the point kinds, each a bit perturbed per beam"""
    ends = [p for k in ("inside", "straddle", "unallocated", "outside", "inside", "straddle") for p in kinds[k]]
    rng = np.random.default_rng(n)
    out = np.zeros((n, 3))
    for i in range(n):
        x, y = ends[i % len(ends)]
        j = rng.uniform(-0.15, 0.15, 2) if i >= len(ends) else (0.0, 0.0)
        out[i, 0], out[i, 1] = (x + j[0] - O) * res, (y + j[1] - O) * res
    return out


def test_match_scenario_covers_every_stencil_kind_and_block_size():
    assert len({match_block(n) for n in BEAMS}) >= 5
    assert {match_block(n) for n in (575, 576, 577)} == {576, 320}
    _, kinds = match_world(0.1)
    for x, y in kinds["straddle"]:
        assert int(math.floor(x)) & 31 == 31 or int(math.floor(y)) & 31 == 31
    for x, y in kinds["inside"]:
        assert int(math.floor(x)) & 31 not in (31,) and int(math.floor(y)) & 31 not in (31,)
    side = MATCH_DEV["dir_dim"] * 32
    assert all(abs(x - O) > side / 2 or abs(y - O) > side / 2 for x, y in kinds["outside"])
    assert all(abs(x - O) < side / 2 - 32 and abs(y - O) < side / 2 - 32 for x, y in kinds["unallocated"])


@pytest.mark.gpu
@pytest.mark.parametrize("res,l2", [(0.1, l2_for(0.1, 63)), (0.025, l2_for(0.025, 63)), (0.025, 0.5), (0.1, 1.0)])
def test_match_across_beam_counts_and_reach(gpu_api, po, res, l2):
    cells, kinds = match_world(res)
    g, o = gpu_api.DynamicDistanceMap(res, l2_max=l2, **MATCH_DEV), po.DDM(res, l2_max=l2)
    g.addObstacle(cells); o.add(cells)
    assert g.update() == o.update()
    rng = np.random.default_rng(3)
    states = np.array([po.se2_from_xyr(0.0, 0.0, 0.0)] + [po.se2_from_xyr(*(rng.uniform(-1, 1, 3) * [3 * res, 3 * res, 0.02])) for _ in range(5)])
    for n in BEAMS:
        s = match_scan(n, res, kinds)
        ne = g.matchNormalEquations(s, states)
        for i, st in enumerate(states):
            assert np.allclose(ne[i, :11], o.match_normal_eq(s, st), rtol=1e-11, atol=1e-13), (n, i)
        if n == 1:   # a one-beam Gauss-Newton system has rank 1: its solve is not compared (the normal equations above are)
            continue
        for strategy in (0, 1):
            sg, stats, _ = g.matchSolve(s, states, strategy=strategy)
            for i, st in enumerate(states):
                sc, _, so = o.match_solve(s, st, strategy=strategy)
                assert np.abs(sg[i] - sc).max() < POSE_TOL, (n, strategy, i)
                assert stats[i, 0] == so[0] and stats[i, 1] == so[1], (n, strategy, i)


def _room_cells(segments, res):
    out = set()
    for x1, y1, x2, y2 in segments:
        n = int(max(abs(x2 - x1), abs(y2 - y1)) / res) + 1
        for k in range(n + 1):
            out.add((cell(x1 + (x2 - x1) * k / n, res), cell(y1 + (y2 - y1) * k / n, res)))
    return np.array(sorted(out), np.uint32)


@pytest.mark.gpu
def test_loc2d_rmse_and_sampling_covariance_at_reach_63(gpu_api, po, synth):
    """Loc2D at 0.1 m with a 63-cell reach: global localization (k_match over 3 000 candidates), RMSE (k_match_error) and the sampling
    covariance (k_sampling)"""
    res = 0.1
    ds = synth.make_dataset("loc_room", 6)
    cells = _room_cells(ds.segments, res)
    kw = dict(trans_thresh=0.01, rot_thresh=0.01, gloc_particles=3000, cov_blend=0.5, resolution=res, l2_max=l2_for(res, 63))
    gl = gpu_api.Loc2D(gpu_api.Loc2D.Options(**kw))
    ol = po.Loc2D(po.LocOptions.defaults(**kw))
    assert gl.distance_map.update() == 0
    gl.distance_map.addObstacle(cells)
    od = ol.dm(); od.add(cells)
    assert gl.distance_map.update() == od.update()
    xs = np.arange(int(-9.9 / res), int(9.9 / res))
    free = np.array([(x + O, y + O) for x in xs[::2] for y in xs[::2]], np.uint32)
    gl.occupancySet(free, -1); gl.occupancySet(cells, 1)
    ol.occ_set(free, -1); ol.occ_set(cells, 1)
    gl.setSeed(77); ol.set_seed(77)
    gl.setPose(0, 0, 0); ol.set_pose(0, 0, 0)
    gl.triggerGlobalLocalization(); ol.trigger_global_localization()
    for t in range(6):
        assert gl.update(ds.scans[t], ds.odom[t], force_update=(t == 0)) == ol.update(ds.scans[t], ds.odom[t], force=(t == 0))
        sc, cov, rmse, _ = ol.get()
        assert np.abs(gl.state() - sc).max() < POSE_TOL, t
        assert abs(gl.getRMSE() - rmse) < 1e-12, t
        assert np.allclose(gl.getCovar(), cov, rtol=1e-8, atol=1e-12), t
        assert gl.globalLocalizationActive() == ol.gloc_active()


# ---- GPU: the filters ------------------------------------------------------------------------------------------------------------------
FILTER_CASES = [(0.025, 1.5), (0.1, 6.0), (0.05, 3.15), (0.03, 0.93)]


def _same_dm(g, o, pa=()):
    n, mn, mx = o.dm_bounds(*pa); w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    _dm_equal(g.exportDistance(*pa, int(mn[0]), int(mn[1]), w, h), o.export_dm(*pa, mn[0], mn[1], w, h), pa)
    ng, mng, mxg = g.mapBounds(*pa, 1)
    assert (mng == mn).all() and (mxg == mx).all()


def _run_slam(gpu_api, po, synth, name, beams, T, res, l2, occupancy=0, **dev):
    ds = synth.make_dataset(name, T, n_beams=beams)
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, resolution=res, l2_max=l2)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(occupancy=occupancy, **kw, **dev))
    o = (po.Slam2DProb if occupancy else po.Slam2D)(po.SlamOptions.defaults(**kw))
    g.setPose(*ds.truth[0]); o.set_pose(*ds.truth[0])
    for t in range(T):
        assert g.update(ds.scans[t], ds.odom[t]) == o.update(ds.scans[t], ds.odom[t]), t
        assert np.abs(g.state() - o.state()).max() < POSE_TOL, t
        cg, _ = g.counters()
        co = o.counters() if occupancy else o.counters()[0]
        assert (cg["evals"], cg["ray_cells"], cg["dm_pops"], cg["gn_iters"]) == (co["evals"], co["ray_cells"], co["dm_pops"], co["gn_iters"]), t
    _same_dm(g, o)
    n, mn, mx = o.occ_bounds(); w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    if occupancy:
        eg, eo = g.exportLogOdds(int(mn[0]), int(mn[1]), w, h), o.export_occ(mn[0], mn[1], w, h)
        assert (eg["prob"] == eo["prob"]).all() and (eg["known"] == eo["known"]).all()
    else:
        eg, eo = g.exportOccupancy(int(mn[0]), int(mn[1]), w, h), o.export_occ(mn[0], mn[1], w, h)
        for k in ("occupied", "visited", "known"):
            assert (eg[k] == eo[k]).all(), k
    return g, o


@pytest.mark.gpu
@pytest.mark.parametrize("occupancy", [0, 1], ids=["frequency", "logodds"])
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
@pytest.mark.parametrize("res,l2", FILTER_CASES)
def test_slam2d_across_reach_equals_oracle(gpu_api, po, synth, monkeypatch, res, l2, form, occupancy):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    _run_slam(gpu_api, po, synth, "room", 360, 10, res, l2, occupancy)


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
@pytest.mark.parametrize("res,l2", FILTER_CASES)
def test_pfslam2d_across_reach_equals_oracle(gpu_api, po, synth, monkeypatch, res, l2, form):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    P, T = 8, 12
    ds = synth.make_dataset("room", T, n_beams=180)
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, seed=5, meas_sigma_gain=0.02, resolution=res, l2_max=l2)
    g = gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(P, pool_slots=16384, **kw))   # fine grids with long waves touch many patches
    o = po.PFSlam2D(po.PFOptions.defaults(P, threads=8, **kw))
    g.setPrior(*ds.truth[0]); o.set_prior(*ds.truth[0])
    n_res = 0
    for t in range(T):
        assert g.update(ds.scans[t], ds.odom[t]) == o.update(ds.scans[t], ds.odom[t]), t
        ro = o.last_resample()
        assert g.lastResample().tolist() == ro.tolist(), t
        n_res += int(len(ro) > 0)
        sg, _ = g.getParticles(); so, _ = o.particles()
        assert np.abs(sg - so).max() < POSE_TOL, t
        if len(ro) == 0:   # on resampling scans the device counts the map work of the set before the resampling (test_gpu_parity.py)
            cg, _ = g.counters(); co, _ = o.counters()
            assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    assert n_res >= 1
    for p in range(P):
        _same_dm(g, o, (p,))


OVERFLOW_DEV = dict(dir_dim=OVERFLOW["dim"], max_beams=OVERFLOW["beams"])


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_slam2d_heap_beyond_shared_memory_equals_oracle(gpu_api, po, synth, monkeypatch, form):
    """the scenario whose lower heap outgrows the 8 192 shared-memory entries (checked on the emulation above): the device carries
    on in global memory and ends with the reference's maps"""
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    c = OVERFLOW
    _run_slam(gpu_api, po, synth, c["name"], c["beams"], c["T"], c["res"], c["l2"], **OVERFLOW_DEV)


# ---- GPU: the global part of the heaps at bench shapes, and overflow -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("l2", [0.5, 1.0])
def test_brushfire_stress_with_a_64_entry_shared_heap(gpu_api, po, monkeypatch, l2):
    """the brushfire parity test with the shared part of each heap shrunk to 64 entries: every update moves its heaps to global memory"""
    import test_gpu_parity
    monkeypatch.setenv("LAMA_BRUSH_SMEM_HEAP", "64")
    test_gpu_parity.test_brushfire_add_remove_stress_bit_exact(gpu_api, po, l2)


@pytest.mark.gpu
def test_slam2d_with_a_64_entry_shared_heap(gpu_api, po, synth, monkeypatch):
    monkeypatch.setenv("LAMA_BRUSH_SMEM_HEAP", "64")
    _run_slam(gpu_api, po, synth, "room", 1080, 12, 0.05, 0.5)


@pytest.mark.gpu
def test_fullsize_run_with_a_64_entry_shared_heap(gpu_api, po, synth, monkeypatch):
    """one of the 256 x 1080 long runs (test_gpu_long.py) with every brushfire heap in global memory after 64 entries"""
    import test_gpu_long
    monkeypatch.setenv("LAMA_BRUSH_SMEM_HEAP", "64")
    test_gpu_long.test_fullsize_long_run_with_resampling(gpu_api, po, synth, monkeypatch, "100000", 60)


@pytest.mark.gpu
def test_heap_overflow_is_reported_with_its_capacity(gpu_api, monkeypatch):
    """a tiny total heap capacity: update() fails with LAMA_ERR_OVERFLOW and the heap's message, never LAMA_OK with a wrong map"""
    monkeypatch.setenv("LAMA_BRUSH_SMEM_HEAP", "16")
    monkeypatch.setenv("LAMA_BRUSH_HEAP_CAP", "64")
    g = gpu_api.DynamicDistanceMap(l2_max=1.0)
    small = np.array([[O + 10, O + 10]], np.uint32)
    g.addObstacle(small)
    with pytest.raises(gpu_api.LamaError) as e:   # one obstacle with a 20-cell reach queues far more than 64 cells
        g.update()
    assert e.value.code == -6 and "heap" in str(e.value) and "64" in str(e.value)


# ---- lama_dm_import checks its cells ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_import_refuses_cells_the_packed_word_cannot_hold(gpu_api, po):
    o = po.DDM(l2_max=1.0)
    o.add(np.array([[O + 40, O + 50], [O + 60, O + 20]], np.uint32))
    o.update()
    e = o.export(O, O, 96, 96)
    g = gpu_api.DynamicDistanceMap(l2_max=1.0)
    g.import_(O, O, e)                                    # what the reference produces is accepted
    _dm_equal(g.export(O, O, 96, 96), e, "import")
    y, x = np.argwhere((e["valid"] == 1) & (e["sqdist"] > 0))[0]
    for field, value in (("sqdist", o.max_sqdist), ("sqdist", 4096), ("ox", 64), ("oy", -65)):
        bad = {k: v.copy() for k, v in e.items()}
        bad[field][y, x] = value
        with pytest.raises(gpu_api.LamaError) as err:
            gpu_api.DynamicDistanceMap(l2_max=1.0).import_(O, O, bad)
        assert err.value.code == -1, (field, value)
    bad = {k: v.copy() for k, v in e.items()}
    inval = np.argwhere((e["known"] == 1) & (e["valid"] == 0))[0]
    bad["sqdist"][inval[0], inval[1]] = o.max_sqdist + 5   # an invalid cell may carry any 12-bit sqdist
    gpu_api.DynamicDistanceMap(l2_max=1.0).import_(O, O, bad)
