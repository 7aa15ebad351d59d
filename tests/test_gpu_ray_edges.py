"""The map update at the edges of the scan geometry, device against oracle, and the 16-bit counter wrap.

The other parity tests cast synthetic room, loop and corridor scans: a few hundred to 1 080 beams in angular order, all shorter
than 30 m, all starting in the sensor cell.  The warp-level code of k_raycast (group-class ballot and its tie, padding lanes, the
per-beam sector shift delta of x-major beams, run merging of equal cells up to a run of 32, the lock step to the longest lane,
the prefetch stop of the strided rounds), the pull form (k_ray_setup / k_ray_pull) and the render (k_render_scans) are driven
here with scans built from wanted map-frame end cells.  Front ends run with max_iter = 0, so every pose is the host-composed
odometry (with PF noise: the host's bit-exact mt19937) and only the cast can differ.

Every scenario has a CPU check (no GPU) that it does what its name says, on the oracle alone.

Counter wrap: FrequencyOccupancyMap::frequency is two independent uint16 (frequency_occupancy_map.h:43-46).  The device packs
them in one word and adds a hit as 0x00010001, so the 65 536th hit of a cell carries into `visited` unless the writer takes
the carry back."""
import math

import numpy as np
import pytest

import global_map_oracle as gmo

O = 1321122 * 32
RES = 0.05
POSE_TOL = 1e-9
WALK, PULL = "0", "100000"   # LAMA_PULL_MAX_PARTICLES: the per-beam walk for every particle count / the pull form for every count


# ---- scan building ------------------------------------------------------------------------------------------------------------
def _quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def scan_to(pose, ends, z=None, origin=(0.0, 0.0, 0.0), quat=(0.0, 0.0, 0.0, 1.0)):
    """sensor-frame points whose beams, cast from the base pose (x, y, theta) through the sensor mount, end at the centres of the
    map cells ends (k, 2); z (k,) world heights of the end points (default: the sensor's height, a planar beam)"""
    e = np.asarray(ends, np.int64).reshape(-1, 2)
    x, y, th = pose
    wx, wy = (e[:, 0] - O) * RES - x, (e[:, 1] - O) * RES - y
    c, s = math.cos(th), math.sin(th)
    base = np.c_[c * wx + s * wy, -s * wx + c * wy, np.full(len(e), origin[2]) if z is None else np.asarray(z, float)]
    return np.ascontiguousarray((base - np.asarray(origin)) @ _quat_matrix(quat))   # R^T (p - origin), row by row


def cell_of(v):
    """Map::w2m of one world coordinate at 0.05 m"""
    return int(np.uint32(v * 20.0 + O + 0.5))


def major_minor(ends, origin):
    d = np.asarray(ends, np.int64) - np.asarray(origin, np.int64)
    return np.abs(d).max(1), np.abs(d[:, 0]) >= np.abs(d[:, 1])


def delta_of(fx, tx):
    """xmajor_seg_shift (ray_core.h): the sector shift of an x-major beam in an x-major group"""
    return ((-fx) if tx < fx else (fx + 1)) & 7


# lengths n = max(|dx|, |dy|) (n - 1 interior cells): 0 (hit in the origin cell), 1, 2, and for every delta and k = 1..3 the
# interior counts 64 k - delta - 1, 64 k - delta, 64 k - delta + 1 around the segment boundaries of the aligned partition
LENGTHS = sorted(set([0, 1, 2] + [64 * k - d + j for d in range(8) for k in (1, 2, 3) for j in (0, 1, 2)]))
OCTANTS = [(xm, sa, sb) for xm in (True, False) for sa in (1, -1) for sb in (1, -1)]


def _beam(o, n, slope, xmajor, sa, sb):
    m = int(n * slope)
    return (o[0] + sa * n, o[1] + sb * m) if xmajor else (o[0] + sb * m, o[1] + sa * n)


OCTANT_LENGTHS = sorted(LENGTHS + [70 + 4 * i for i in range(31)])   # 64 beams: two whole groups per octant, few short ones
assert len(OCTANT_LENGTHS) == 64


def edge_groups(o):
    """the end cells of one edge scan from origin cell o, as a list of (name, ends) blocks: each block is one 32-beam group of the
    scan, the last one has 7 beams (25 padding lanes)"""
    blocks = []
    for xm, sa, sb in OCTANTS:   # every length in every octant, each on its own line: slope i / 63 from axis-aligned to exactly diagonal
        ends = [_beam(o, n, i / 63, xm, sa, sb) for i, n in enumerate(OCTANT_LENGTHS)]
        for g0 in range(0, len(ends), 32):
            blocks.append((f"octant {'x' if xm else 'y'}{sa:+d}{sb:+d}", ends[g0:g0 + 32]))
    long_ = [100 + 3 * i for i in range(16)]
    xs = [_beam(o, n, 0.3, True, 1, 1) for n in long_]
    ys = [_beam(o, n, 0.3, False, -1, 1) for n in long_]
    blocks.append(("tie 16/16 (y-major group)", [b for pair in zip(xs, ys) for b in pair]))
    xs17 = [_beam(o, 120 + 4 * i, 0.2, True, -1, -1) for i in range(17)]
    ys15 = [_beam(o, 130 + 4 * i, 0.4, False, 1, -1) for i in range(15)]
    blocks.append(("17/15 (x-major group, strided y-major minority)", (xs17 + ys15)[::-1]))
    xs15 = [_beam(o, 90 + 5 * i, 0.1, True, 1, -1) for i in range(15)]
    ys17 = [_beam(o, 95 + 5 * i, 0.6, False, 1, 1) for i in range(17)]
    blocks.append(("15/17", [b for k in range(17) for b in ([ys17[k]] + ([xs15[k]] if k < 15 else []))]))
    blocks.append(("run of 32, y-major", [_beam(o, 150, 0.25, False, 1, 1)] * 32))
    blocks.append(("run of 32, x-major", [_beam(o, 170, 0.25, True, -1, 1)] * 32))
    a, b = _beam(o, 140, 0.7, True, 1, -1), _beam(o, 141, 0.7, True, 1, -1)
    blocks.append(("alternating end cells", [a, b] * 16))
    blocks.append(("padding lanes", [_beam(o, 60 + 11 * i, 0.45, i % 2 == 0, 1 if i < 4 else -1, 1) for i in range(7)]))
    return blocks


def edge_ends(o, shuffle_seed=None):
    ends = np.array([e for _, b in edge_groups(o) for e in b], np.int64)
    if shuffle_seed is not None:
        ends = ends[np.random.default_rng(shuffle_seed).permutation(len(ends))]
    return ends


def group_classes(ends, o):
    """group_is_xmajor of every 32-beam group (planar beams; the tie goes to y-major) and its x-major / planar counts"""
    out = []
    n, xm = major_minor(ends, o)
    for g0 in range(0, len(ends), 32):
        nx = int(xm[g0:g0 + 32].sum())
        out.append((2 * nx > len(xm[g0:g0 + 32]), nx, len(xm[g0:g0 + 32])))
    return out


# ---- scenario: a Slam2D / PFSlam2D sequence of edge scans -------------------------------------------------------------------------
X0, Y0 = 0.0, 0.0   # the prior: cell (O, O)
# the walk logs every touch of a candidate cell (hit in this scan or a distance-map obstacle); edge scans cross many of them, so the
# engines get a 16 384-record log (3 * max_beams, rounded up to a power of two), which fits shared memory with a 32-patch window
EDGE_DEV = dict(dir_dim=32, max_beams=4096)
# every end cell of an edge scan is a separate new obstacle: a one-cell distance-map reach keeps these tests about the ray cast
# (test_gpu_reach.py covers reaches up to 63 cells and brushfire heaps that outgrow shared memory)
EDGE_L2 = dict(l2_max=0.05)


def edge_sequence():
    """(odometry reading, base pose, end cells) per scan: 8 scans stepping the origin one cell in +x (every x mod 8, so every delta in
    both x directions), the fourth one in a shuffled beam order; then 5 scans turning in place that shoot through the walls of
    the last edge scan (end offsets doubled: the doubled Bresenham line passes the old end cell) -- misses on obstacle cells
    in x-major strided segments, which must end in removeObstacle"""
    seq = []
    for s in range(8):
        o = (O + s, O)
        seq.append(((s * RES, 0.0, 0.0), (X0 + s * RES, Y0, 0.0), edge_ends(o, shuffle_seed=5 if s == 3 else None)))
    o = (O + 7, O)
    ends = edge_ends(o)
    # beams up to 97 cells long are doubled (they stay inside the edge scan's area, so the candidate patches stay within the walk's
    # 192 bitmaps); longer beams hit their old cells again
    n, _ = major_minor(ends, o)
    through = np.where((n <= 97)[:, None], (ends - np.array(o)) * 2 + np.array(o), ends)
    for r in range(1, 6):
        seq.append(((7 * RES, 0.0, 0.02 * r), (X0 + 7 * RES, Y0, 0.02 * r), through))
    return seq


def _run_oracle_slam(po, seq, **kw):
    o = po.Slam2D(po.SlamOptions.defaults(trans_thresh=0.01, rot_thresh=0.01, max_iter=0, **kw))
    o.set_pose(X0, Y0, 0.0)
    return o


def _obstacles(dm):
    return set(zip(*np.nonzero((dm["valid"] == 1) & (dm["sqdist"] == 0))))


# ---- CPU: the scenarios do what their names say ----------------------------------------------------------------------------------
def test_edge_scans_cover_every_delta_length_and_group_class():
    seq = edge_sequence()
    deltas = set()
    for _, pose, ends in seq[:8]:
        o = (cell_of(pose[0]), cell_of(pose[1]))
        n, xm = major_minor(ends, o)
        for (tx, _), nn, x in zip(ends, n, xm):
            if x and nn >= 2:
                deltas.add((tx > o[0], delta_of(o[0], tx)))
        assert set(LENGTHS) <= set(n.tolist())
    assert deltas == {(d, k) for d in (True, False) for k in range(8)}           # every delta in both x directions
    for d in range(8):                                                           # the interior counts around every shifted boundary
        assert all(64 * k - d + j in LENGTHS for k in (1, 2, 3) for j in (0, 1, 2))
    o = (O, O)
    blocks = dict(edge_groups(o))
    classes = group_classes(np.array([e for _, b in edge_groups(o) for e in b]), o)
    assert [len(b) for _, b in edge_groups(o)][:-1] == [32] * (len(edge_groups(o)) - 1)   # every named block is one group
    assert len(edge_ends(o)) % 32 == 7                                          # the last group has padding lanes
    names = [nm for nm, _ in edge_groups(o)]
    by_name = {nm: classes[i] for i, nm in enumerate(names)}
    assert by_name["tie 16/16 (y-major group)"] == (False, 16, 32)
    assert by_name["17/15 (x-major group, strided y-major minority)"] == (True, 17, 32)
    assert by_name["15/17"] == (False, 15, 32)
    n, _ = major_minor(blocks["17/15 (x-major group, strided y-major minority)"], o)
    assert n.min() > 64                                                          # the minority reaches the strided rounds
    assert len(set(map(tuple, blocks["run of 32, y-major"]))) == 1 and len(set(map(tuple, blocks["alternating end cells"]))) == 2
    for xm, sa, sb in OCTANTS:                                                   # axis-aligned and exact diagonals in all 8 octants
        ends = np.array([e for nm, b in edge_groups(o) if nm == f"octant {'x' if xm else 'y'}{sa:+d}{sb:+d}" for e in b]) - np.array(o)
        assert ((ends[:, 0] == 0) | (ends[:, 1] == 0)).any() and (np.abs(ends[:, 0]) == np.abs(ends[:, 1])).any()
    assert any(c[0] for c in classes) and any(not c[0] for c in classes)
    assert (edge_ends(o, 5) != edge_ends(o)).any() and sorted(map(tuple, edge_ends(o, 5))) == sorted(map(tuple, edge_ends(o)))


def test_edge_sequence_poses_are_the_odometry_and_the_walls_are_removed(po):
    """max_iter = 0: every pose is the composed odometry (the end cells are where they were aimed); the through-the-walls scans
    remove obstacles of the last edge scan; every beam ends in the cell it was built for"""
    seq = edge_sequence()
    o = _run_oracle_slam(po, seq)
    obst = []
    for t, (odom, pose, ends) in enumerate(seq):
        assert o.update(scan_to(pose, ends), odom)
        st = o.state()
        assert abs(st[2] - pose[0]) < 1e-12 and abs(st[3] - pose[1]) < 1e-12 and abs(math.atan2(st[1], st[0]) - pose[2]) < 1e-12
        if t == 0:   # every beam ends in the cell it was aimed at: each end cell holds at least its hits
            n, mn, mx = o.occ_bounds()
            occ = o.export_occ(mn[0], mn[1], int(mx[0] - mn[0]), int(mx[1] - mn[1]))
            cells, hits = np.unique(ends, axis=0, return_counts=True)
            assert (occ["occupied"][cells[:, 1] - mn[1], cells[:, 0] - mn[0]] >= hits).all()
        n, mn, mx = o.dm_bounds()
        dm = o.export_dm(mn[0], mn[1], int(mx[0] - mn[0]), int(mx[1] - mn[1]))
        obst.append({(int(y) + int(mn[1]), int(x) + int(mn[0])) for y, x in _obstacles(dm)})
    removed = obst[7] - obst[-1]
    assert len(removed) > 10                                                     # removeObstacle fired on walls of the edge scan
    assert len(removed & {(int(e[1]), int(e[0])) for e in seq[7][2]}) > 10        # ... the end cells its beams were aimed at


# ---- GPU: edge scans through Slam2D and PFSlam2D ----------------------------------------------------------------------------------
def _same_maps(g, o, particle=None):
    pa = () if particle is None else (particle,)
    for kind, ob in ((0, o.occ_bounds), (1, o.dm_bounds)):
        n, mn, mx = ob(*pa)
        ng, mng, mxg = g.mapBounds(*pa, kind)
        assert (mng == mn).all() and (mxg == mx).all(), (particle, kind)          # Map::bounds
        if kind == 0:
            assert ng == n
    n, mn, mx = o.occ_bounds(*pa); w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g.exportOccupancy(*pa, int(mn[0]), int(mn[1]), w, h), o.export_occ(*pa, mn[0], mn[1], w, h)
    for k in ("occupied", "visited", "known"):
        assert (a[k] == b[k]).all(), (particle, k, int((a[k] != b[k]).sum()))
    n, mn, mx = o.dm_bounds(*pa); w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g.exportDistance(*pa, int(mn[0]), int(mn[1]), w, h), o.export_dm(*pa, mn[0], mn[1], w, h)
    for k in ("sqdist", "valid", "ox", "oy", "queued", "known"):
        assert (a[k] == b[k]).all(), (particle, k, int((a[k] != b[k]).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [{}, dict(truncated_ray=1.0), dict(truncated_range=4.0), dict(truncated_ray=1.5, truncated_range=6.0)],
                         ids=["plain", "truncated_ray", "truncated_range", "both"])
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_slam2d_edge_scans_equal_oracle(gpu_api, po, monkeypatch, form, opts):
    """per scan: update() return value, ray_cells, dm_pops; at the end every occupancy and distance cell and both map bounds.
    truncated_ray moves every beam's start (a different delta per beam of one group; the pull form hands such scans to the walk)"""
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    seq = edge_sequence()
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(trans_thresh=0.01, rot_thresh=0.01, max_iter=0, **EDGE_DEV, **EDGE_L2, **opts))
    g.setPose(X0, Y0, 0.0)
    o = _run_oracle_slam(po, seq, **EDGE_L2, **opts)
    for t, (odom, pose, ends) in enumerate(seq):
        s = scan_to(pose, ends)
        assert g.update(s, odom) == o.update(s, odom), t
        cg, _ = g.counters(); co, _ = o.counters()
        assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    assert np.abs(g.state() - o.state()).max() < POSE_TOL
    _same_maps(g, o)


def _pf_pair(gpu_api, po, P, dev=None, **kw):
    opts = dict(trans_thresh=0.01, rot_thresh=0.01, max_iter=0, **kw)
    g = gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(P, **opts, **(dev or {})))
    o = po.PFSlam2D(po.PFOptions.defaults(P, threads=4, **opts))
    g.setPrior(X0, Y0, 0.0); o.set_prior(X0, Y0, 0.0)
    return g, o


def _pf_step(g, o, s, odom, t):
    assert g.update(s, odom) == o.update(s, odom), t
    ro = o.last_resample()
    assert g.lastResample().tolist() == ro.tolist(), t
    sg, _ = g.getParticles(); so, _ = o.particles()
    assert np.abs(sg - so).max() < POSE_TOL, t
    if len(ro) == 0:   # on resampling scans the device counts the map work of the set before the resampling (test_gpu_parity.py)
        cg, _ = g.counters(); co, _ = o.counters()
        assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    return so


def test_pf_edge_scan_origins_spread_over_sub_cell_positions(po):
    """the PF's odometry noise puts the particles' ray starts at different cells: several x mod 8 (so several delta) in one launch"""
    seq = edge_sequence()
    o = po.PFOptions.defaults(8, trans_thresh=0.01, rot_thresh=0.01, max_iter=0, seed=17, threads=4)
    pf = po.PFSlam2D(o)
    pf.set_prior(X0, Y0, 0.0)
    xs = set()
    for odom, pose, ends in seq[:4]:
        pf.update(scan_to(pose, ends), odom)
        st, _ = pf.particles()
        xs |= {cell_of(v) % 8 for v in st[:, 2]}
    assert len(xs) >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_pfslam2d_edge_scans_equal_oracle(gpu_api, po, monkeypatch, form):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    P = 8
    g, o = _pf_pair(gpu_api, po, P, seed=17, dev=EDGE_DEV, **EDGE_L2)
    for t, (odom, pose, ends) in enumerate(edge_sequence()):
        _pf_step(g, o, scan_to(pose, ends), odom, t)
    for p in range(P):
        _same_maps(g, o, p)


# ---- beam counts, the window's edges and overflow ---------------------------------------------------------------------------------
BEAM_COUNTS = (1, 2, 31, 32, 33, 63, 65, 513, 1081, 4096, 4097)   # 4096 = kPullMaxBeams: above it the pull form hands the scan to the walk
SIDE = 16 * 32                                                    # cells per side of a dir_dim = 16 window centred on the prior (0, 0)
W0 = O - SIDE // 2                                                # its first cell


def count_ends(n, o=(O, O)):
    """n beams in angular order to a ring of cells 200 away (inside the 16-patch window around its centre).  A ray crosses few other
    end cells, so the walk's touch log holds the candidate touches of 4 097 beams"""
    ang = (np.arange(n) + 0.5) * (2 * math.pi / n) + 0.1 * n
    return np.c_[o[0] + np.round(200 * np.cos(ang)), o[1] + np.round(200 * np.sin(ang))].astype(np.int64)


def corner_ends():
    """from the window's cell (1, 1): the opposite cell (side - 2, side - 2), and cells at 1 and side - 2 along both edges (the
    obstacles' one-cell distance-map reach stays inside the window)"""
    first, last = W0 + 1, W0 + SIDE - 2
    return np.array([(last, last), (last, first), (first, last), (last, first + 1), (first + 1, last), (last, last - 1)] * 11, np.int64)


def beam_count_sequence():
    seq = [((0.0, 0.0, 0.02 * i), (X0, Y0, 0.02 * i), count_ends(n)) for i, n in enumerate(BEAM_COUNTS)]
    cx = (W0 + 1 - O) * RES                                      # the window's cell (1, 1) as the base pose
    seq.append(((cx, cx, 0.0), (cx, cx, 0.0), corner_ends()))
    return seq


def test_beam_count_and_corner_scenario():
    seq = beam_count_sequence()
    assert [len(e) for _, _, e in seq[:-1]] == list(BEAM_COUNTS)
    for _, pose, ends in seq[:-1]:
        assert ends.min() >= W0 and ends.max() < W0 + SIDE
    _, pose, ends = seq[-1]
    assert (cell_of(pose[0]), cell_of(pose[1])) == (W0 + 1, W0 + 1)
    assert ends.max() == W0 + SIDE - 2 and ends.min() == W0 + 1
    assert max(major_minor(ends, (W0 + 1, W0 + 1))[0]) == SIDE - 3              # corner to corner


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_beam_counts_and_window_corners_equal_oracle(gpu_api, po, monkeypatch, form):
    """scans of 1 .. 4 097 beams in a 16-patch window, then a corner-to-corner scan across it"""
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(trans_thresh=0.01, rot_thresh=0.01, max_iter=0, dir_dim=16, max_beams=4097, **EDGE_L2))
    g.setPose(X0, Y0, 0.0)
    o = _run_oracle_slam(po, None, **EDGE_L2)
    for t, (odom, pose, ends) in enumerate(beam_count_sequence()):
        s = scan_to(pose, ends)
        assert g.update(s, odom) == o.update(s, odom), t
        cg, _ = g.counters(); co, _ = o.counters()
        assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    _same_maps(g, o)


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_beam_one_cell_past_the_window_is_an_error(gpu_api, monkeypatch, form):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(trans_thresh=0.01, rot_thresh=0.01, max_iter=0, dir_dim=16, **EDGE_L2))
    g.setPose(X0, Y0, 0.0)
    g.update(scan_to((X0, Y0, 0.0), [(W0 + SIDE - 2, O), (W0 + 1, O)]), (0.0, 0.0, 0.0))   # obstacles and their reach inside: fine
    with pytest.raises(gpu_api.LamaError) as e:
        g.update(scan_to((X0, Y0, 0.02), [(W0 + SIDE, O)]), (0.0, 0.0, 0.02))
    assert e.value.code == -4


@pytest.mark.gpu
def test_render_beam_one_cell_past_the_window_is_an_error(gpu_api):
    g = gpu_api.FrequencyOccupancyMap(RES, dir_dim=16)
    ident = np.array([[1.0, 0.0, 0.0, 0.0]])
    g.insertScans([scan_to((0.0, 0.0, 0.0), [(W0 + SIDE - 1, W0)])], ident, full=True)
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertScans([scan_to((0.0, 0.0, 0.0), [(O, W0 - 1)])], ident, full=True)
    assert e.value.code == -4


# ---- a tilted sensor with planar and non-planar beams interleaved in one group -----------------------------------------------------
TILT_ORIGIN = (0.1, 0.0, 0.3)
TILT_QUAT = (0.0, math.sin(0.025), 0.0, math.cos(0.025))


def tilted_scan(pose):
    o = (cell_of(pose[0] + TILT_ORIGIN[0]), cell_of(pose[1]))
    ends = edge_ends(o)
    z = np.where(np.arange(len(ends)) % 3 == 1, TILT_ORIGIN[2] + 0.4, TILT_ORIGIN[2])   # every third beam leaves the sensor's z cell
    return scan_to(pose, ends, z=z, origin=TILT_ORIGIN, quat=TILT_QUAT), z


def test_tilted_scan_mixes_planar_and_non_planar_beams_in_each_group():
    pts, z = tilted_scan((X0, Y0, 0.0))
    R = _quat_matrix(TILT_QUAT)
    world_z = pts @ R.T[:, 2] + TILT_ORIGIN[2]
    zc = np.array([cell_of(v) for v in world_z])
    planar = zc == cell_of(TILT_ORIGIN[2])
    assert (planar == (z == TILT_ORIGIN[2])).all()
    for g0 in range(0, len(planar) - 31, 32):
        assert 0 < planar[g0:g0 + 32].sum() < 32


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_tilted_sensor_mixed_beams_equal_oracle(gpu_api, po, monkeypatch, form):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    g, o = _pf_pair(gpu_api, po, 4, seed=23, dev=EDGE_DEV, **EDGE_L2)
    for t in range(4):
        pose = (X0 + t * RES, Y0, 0.0)
        s, _ = tilted_scan(pose)
        odom = (t * RES, 0.0, 0.0)
        assert g.update(s, odom, origin=TILT_ORIGIN, quat=TILT_QUAT) == o.update(s, odom, origin=TILT_ORIGIN, quat=TILT_QUAT), t
        cg, _ = g.counters(); co, _ = o.counters()
        if len(o.last_resample()) == 0:
            assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    for p in range(4):
        _same_maps(g, o, p)


# ---- the render ------------------------------------------------------------------------------------------------------------------
def _render_edge_inputs():
    scans, states, origins, quats = [], [], [], []
    for s in range(8):
        pose = ((-3 + s) * RES * 3 + 0.013 * s, 0.4 - 0.021 * s, 0.0)   # origins at several x mod 8 and sub-cell positions
        o = (cell_of(pose[0]), cell_of(pose[1]))
        scans.append(scan_to(pose, edge_ends(o, shuffle_seed=9 if s == 5 else None)))
        states.append([1.0, 0.0, pose[0], pose[1]])
        origins.append([0.0, 0.0, 0.0]); quats.append([0.0, 0.0, 0.0, 1.0])
    s, _ = tilted_scan((0.2, -0.3, 0.0))
    scans.append(s); states.append([1.0, 0.0, 0.2, -0.3]); origins.append(list(TILT_ORIGIN)); quats.append(list(TILT_QUAT))
    return scans, np.array(states), np.array(origins), np.array(quats)


@pytest.mark.gpu
def test_render_edge_scans_equal_oracle(gpu_api):
    from test_global_map import _same_map
    scans, states, origins, quats = _render_edge_inputs()
    g = gpu_api.FrequencyOccupancyMap(RES)
    o = gmo.OccupancyMap(RES)
    for full in (True, False, True):
        assert g.insertScans(scans, states, full=full, origins=origins, quats=quats) == o.insert_scans(scans, states, full, origins=origins, quats=quats)
        _same_map(g, o)


# ---- the 16-bit counter wrap -------------------------------------------------------------------------------------------------------
# Turning in place keeps the sensor cell S = (O, O) fixed.  Every scan: 880 beams end in C, 200 end in D, a cell on the common
# ray S -> C, so C takes 880 hits (occupied and visited wrap after 75 scans: a packed hit carries into visited), D 200 hits and
# 880 misses, and the cells of the common ray before D 1 080 misses (visited wraps after 61 scans, through 32-lane run merges).
# D stays free (4 * 200 < 1 080) until its visited wraps; the first touch after the wrap to 0 is a hit, so D becomes occupied only
# because visited wrapped, and the wrap itself calls addObstacle.
WRAP_SCANS = 80
WRAP_C = (O + 10, O + 5)


def _ray_cells(a, b):
    """Map::computeRay's interior cells (planar)"""
    dx, dy = b[0] - a[0], b[1] - a[1]
    n = max(abs(dx), abs(dy))
    out = []
    for i in range(1, n):
        out.append((a[0] + (1 if dx >= 0 else -1) * ((2 * i * abs(dx) + n) // (2 * n)), a[1] + (1 if dy >= 0 else -1) * ((2 * i * abs(dy) + n) // (2 * n))))
    return out


WRAP_D = _ray_cells((O, O), WRAP_C)[6]


def wrap_targets():
    """per beam: True = ends in D.  Beams 736 .. 935 end in D, all others in C: groups 0 .. 22 are 32 identical beams (one run of
    32 on every cell of the common ray), and in scan 61 D's visited count (1 080 * 60 before it) reaches 0 after the misses of
    beams 0 .. 735, so the next touch is a hit."""
    first_after = 65536 - 1080 * 60
    d = np.zeros(1080, bool)
    d[first_after:first_after + 200] = True
    return d


def wrap_scan(theta, ends_mask=None):
    d = wrap_targets() if ends_mask is None else ends_mask
    ends = np.where(d[:, None], np.array(WRAP_D), np.array(WRAP_C))
    return scan_to((X0, Y0, theta), ends)


def wrap_odom(t):
    return (0.0, 0.0, 0.03 * t)


def test_wrap_scenario_wraps_the_oracle_counters_and_the_wrap_adds_an_obstacle(po):
    o = _run_oracle_slam(po, None)
    d_obstacle = []
    for t in range(WRAP_SCANS):
        assert o.update(wrap_scan(0.03 * t), wrap_odom(t))
        st = o.state()
        assert abs(st[2]) < 1e-12 and abs(st[3]) < 1e-12 and abs(math.atan2(st[1], st[0]) - 0.03 * t) < 1e-12
        dm = o.export_dm(WRAP_D[0], WRAP_D[1], 1, 1)
        d_obstacle.append(bool(dm["valid"][0, 0] and dm["sqdist"][0, 0] == 0))
    occ = o.export_occ(O, O, 16, 8)
    cx, cy = WRAP_C[0] - O, WRAP_C[1] - O
    assert (int(occ["occupied"][cy, cx]), int(occ["visited"][cy, cx])) == ((880 * WRAP_SCANS) & 0xFFFF,) * 2
    assert 880 * WRAP_SCANS > 65536                                                       # C's occupied wrapped
    dx, dy = WRAP_D[0] - O, WRAP_D[1] - O
    assert (int(occ["occupied"][dy, dx]), int(occ["visited"][dy, dx])) == (200 * WRAP_SCANS, (1080 * WRAP_SCANS) & 0xFFFF)
    ray = _ray_cells((O, O), WRAP_D)
    x, y = ray[2]
    assert int(occ["visited"][y - O, x - O]) == (1080 * WRAP_SCANS) & 0xFFFF and occ["occupied"][y - O, x - O] == 0
    assert not any(d_obstacle[:60]) and d_obstacle[60] and d_obstacle[-1]              # D turned obstacle in the wrap scan
    assert WRAP_D in _ray_cells((O, O), WRAP_C) and WRAP_D not in (WRAP_C, (O, O))


def _wrap_region(g, o, particle=None):
    pa = () if particle is None else (particle,)
    a, b = g.exportOccupancy(*pa, O - 2, O - 2, 20, 12), o.export_occ(*pa, O - 2, O - 2, 20, 12)
    for k in ("occupied", "visited", "known"):
        assert (a[k] == b[k]).all(), (particle, k, [(int(x) + O - 2, int(y) + O - 2, int(a[k][y, x]), int(b[k][y, x])) for y, x in zip(*np.nonzero(a[k] != b[k]))][:4])


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_slam2d_counter_wrap_equals_oracle(gpu_api, po, monkeypatch, form):
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(trans_thresh=0.01, rot_thresh=0.01, max_iter=0))
    g.setPose(X0, Y0, 0.0)
    o = _run_oracle_slam(po, None)
    for t in range(WRAP_SCANS):
        s = wrap_scan(0.03 * t)
        assert g.update(s, wrap_odom(t)) == o.update(s, wrap_odom(t)), t
        cg, _ = g.counters(); co, _ = o.counters()
        assert (cg["ray_cells"], cg["dm_pops"]) == (co["ray_cells"], co["dm_pops"]), t
    _wrap_region(g, o)
    _same_maps(g, o)


@pytest.mark.gpu
@pytest.mark.parametrize("form", [WALK, PULL], ids=["walk", "pull"])
def test_pfslam2d_counter_wrap_equals_oracle(gpu_api, po, monkeypatch, form):
    """the same scans through 4 particles whose odometry noise is far below a cell: every particle's C wraps"""
    monkeypatch.setenv("LAMA_PULL_MAX_PARTICLES", form)
    P = 4
    g, o = _pf_pair(gpu_api, po, P, seed=29, srr=1e-6, str=1e-6, stt=1e-6, srt=1e-6)
    for t in range(WRAP_SCANS):
        so = _pf_step(g, o, wrap_scan(0.03 * t), wrap_odom(t), t)
    assert np.abs(so[:, 2:]).max() < 0.01                       # every particle still in the sensor cell
    for p in range(P):
        _wrap_region(g, o, p)
        _same_maps(g, o, p)


def _wrap_render_inputs(counts):
    scans, states = [], []
    for k, n in enumerate(counts):
        th = 0.03 * k
        scans.append(wrap_scan(th, np.zeros(1080, bool))[:n])       # every beam ends in C
        states.append([math.cos(th), math.sin(th), 0.0, 0.0])
    return scans, np.array(states)


def test_wrap_render_inputs_touch_c_as_planned():
    o = gmo.OccupancyMap(RES)
    scans, states = _wrap_render_inputs([1080] * 60 + [736])
    o.insert_scans(scans, states, True)
    e = o.export(O, O, 16, 8)
    cx, cy = WRAP_C[0] - O, WRAP_C[1] - O
    assert sum(len(s) for s in scans) == 65536
    assert (int(e["occupied"][cy, cx]), int(e["visited"][cy, cx]), int(e["known"][cy, cx])) == (0, 0, 1)   # exactly 2^16 hits


@pytest.mark.gpu
def test_render_counter_wrap_equals_oracle(gpu_api):
    """62 scans of 1 080 beams into C in one insertScans call: occupied and visited of C and visited of the common ray wrap"""
    from test_global_map import _same_map
    scans, states = _wrap_render_inputs([1080] * 62)
    g, o = gpu_api.FrequencyOccupancyMap(RES), gmo.OccupancyMap(RES)
    assert g.insertScans(scans, states, full=True) == o.insert_scans(scans, states, True)
    _same_map(g, o)


@pytest.mark.gpu
def test_render_touching_a_cell_exactly_65536_times(gpu_api):
    """C takes exactly 2^16 hits and the cells of its ray exactly 2^16 misses in one render: their counters come back to {0, 0}.
    The device sets the known plane of a render from `word != 0`, so these cells -- and only these -- are not marked known
    (DESIGN.md section 10); every counter is exact"""
    scans, states = _wrap_render_inputs([1080] * 60 + [736])
    g, o = gpu_api.FrequencyOccupancyMap(RES), gmo.OccupancyMap(RES)
    assert g.insertScans(scans, states, full=True) == o.insert_scans(scans, states, True)
    ng, mn, mx = g.bounds()
    no, mn2, mx2 = o.bounds()
    assert ng == no and (mn == mn2).all() and (mx == mx2).all()
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g.export(int(mn[0]), int(mn[1]), w, h), o.export(int(mn[0]), int(mn[1]), w, h)
    assert (a["occupied"] == b["occupied"]).all() and (a["visited"] == b["visited"]).all()
    full_turn = {WRAP_C} | set(_ray_cells((O, O), WRAP_C))
    differ = {(int(x) + int(mn[0]), int(y) + int(mn[1])) for y, x in zip(*np.nonzero(a["known"] != b["known"]))}
    assert differ == full_turn
    for x, y in full_turn:
        assert b["known"][y - mn[1], x - mn[0]] == 1 and a["known"][y - mn[1], x - mn[0]] == 0 and b["visited"][y - mn[1], x - mn[0]] == 0
