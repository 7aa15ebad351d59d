"""Every 2-D map reader while the moving window has parked patches: distance() (bilinear stencils whose corners lie partly in the
window and partly in parked patches), occupancyQuery() (log-odds `known` bit included), exportImage(), exportLogOdds() and .sdm files,
on frequency and log-odds Slam2D (a transient map among them) and PFSlam2D particles (resampled copies of parked lists included),
compared with the oracle's maps, which have no edge, and with an independent float64 bilinear reference.  LidarOdometry2D, whose
transient map never leaves a patch parked, is compared after its window has moved.  Also the scan correlation while patches are
parked: exact inside the window, a loud LAMA_ERR_WINDOW when it reaches parked ground."""
import tempfile

import numpy as np
import pytest

from iris_lama_b200 import sdm
from test_gpu_window_follow import POSE_TOL, _close, _out_and_back
from test_sdm_io import _same_files

pytestmark = pytest.mark.gpu

RES = 0.05
SCALE = 1.0 / RES
PATCH = 32
UC = sdm.UNIVERSAL_CONSTANT
OFFSET = float((UC >> 1) * PATCH)           # Map::w2m's offset in cells (map.cpp:55-58)
PARKED_SHARE = 0.2                          # least share of the probe's distance stencils that must reach a parked patch
CELL_SHARE = 0.1                            # and of its occupancy cells (whole rows along the window's mostly unmapped edges among them)
EDGE_OFFSETS = np.arange(-2.0, 2.01, 0.5)   # cells from a window edge: every stencil that straddles it
FAR = np.array([(1000.0, 1000.0), (-800.0, 5.0), (3.0, -900.0), (2000.0, -2000.0)])


def _pid(cx, cy):
    return (np.asarray(cx, np.int64) >> 5) * UC + (np.asarray(cy, np.int64) >> 5)


def _world(m):
    return (np.asarray(m, np.float64) - OFFSET) / SCALE


def _patches(f):
    """(px, py) arrays of the patches of a read .sdm file"""
    ids = np.array(sorted(f["patches"]), np.int64)
    return ids // UC, ids % UC


def _probe_points(win, dm_px, dm_py, parked_ids, rng):
    """world points (n, 3): both sides of the four window edges, both sides of every parked patch's edges, every patch of the map's
    bounds grown by two patches, uniform points over that box, and a few far from anything mapped"""
    lo = np.array([dm_px.min(), dm_py.min()]) * PATCH
    hi = (np.array([dm_px.max(), dm_py.max()]) + 1) * PATCH
    glo, ghi = lo - 2 * PATCH, hi + 2 * PATCH
    bx, by, dim = win["base"][0], win["base"][1], win["dim"]
    pts = []
    for axis, edges in ((0, (bx * PATCH, (bx + dim) * PATCH)), (1, (by * PATCH, (by + dim) * PATCH))):
        along = np.linspace(lo[1 - axis] - PATCH, hi[1 - axis] + PATCH, 48) + rng.uniform(0, 1, 48)
        for e in edges:
            for off in EDGE_OFFSETS:
                m = np.empty((48, 2))
                m[:, axis] = e + off
                m[:, 1 - axis] = along
                pts.append(m)
    ppx, ppy = parked_ids // UC, parked_ids % UC
    k = max(4, int(np.ceil(3000 / (8 * max(1, len(parked_ids))))))
    for px, py in zip(ppx, ppy):
        for axis in (0, 1):
            e0 = (px, py)[axis] * PATCH
            for e in (e0 - 0.5, e0 + 0.5, e0 + PATCH - 0.5, e0 + PATCH + 0.5):
                m = np.empty((k, 2))
                m[:, axis] = e
                m[:, 1 - axis] = (py, px)[axis] * PATCH + rng.uniform(0, PATCH, k)
                pts.append(m)
    gx, gy = np.meshgrid(np.arange(glo[0], ghi[0], PATCH), np.arange(glo[1], ghi[1], PATCH))
    corners = np.c_[gx.ravel(), gy.ravel()].astype(np.float64)
    pts += [corners + PATCH / 2 + 0.25, corners + rng.uniform(0, PATCH, corners.shape)]
    pts.append(rng.uniform(glo, ghi, (1500, 2)))
    m = np.concatenate(pts)
    w = np.c_[_world(m), np.zeros(len(m))]
    return np.concatenate([w, np.c_[FAR, np.zeros(len(FAR))]])


def _bilinear_reference(po, dm_handle, pts, glo, ghi):
    """float64 DynamicDistanceMap::distance (dynamic_distance_map.cpp:66-92) from the oracle's exported cells: an absent or invalid
    corner is max_sqdist away"""
    max_sq = po.DDM(handle=dm_handle.value).max_sqdist
    dmax = np.sqrt(float(max_sq)) * RES
    x0, y0 = int(glo[0]) - 1, int(glo[1]) - 1
    w, h = int(ghi[0] - glo[0]) + 2, int(ghi[1] - glo[1]) + 2
    e = po._export_dm(po.lib().orc_ddm_export, (dm_handle,), x0, y0, w, h)
    grid = np.where(e["valid"] != 0, np.sqrt(e["sqdist"].astype(np.float64)) * RES, dmax)
    m = pts[:, :2] * SCALE + OFFSET
    d = np.floor(m).astype(np.int64)
    mu = m - d

    def v(cx, cy):
        out = np.full(len(cx), dmax)
        inside = (cx >= x0) & (cx < x0 + w) & (cy >= y0) & (cy < y0 + h)
        out[inside] = grid[cy[inside] - y0, cx[inside] - x0]
        return out

    v0, v1, v2, v3 = v(d[:, 0], d[:, 1]), v(d[:, 0] + 1, d[:, 1]), v(d[:, 0], d[:, 1] + 1), v(d[:, 0] + 1, d[:, 1] + 1)
    nu0, nu1 = 1.0 - mu[:, 0], 1.0 - mu[:, 1]
    dist = v0 * nu0 * nu1 + v1 * nu1 * mu[:, 0] + v2 * nu0 * mu[:, 1] + v3 * mu[:, 0] * mu[:, 1]
    gx = -((v0 - v1) * nu1 + (v2 - v3) * mu[:, 1]) * SCALE
    gy = -((v0 - v2) * nu0 + (v1 - v3) * mu[:, 0]) * SCALE
    return dist, np.c_[gx, gy, np.zeros(len(gx))], d, dmax


def _logodds_from_file(f, x0, y0, w, h):
    """(prob, known) of a log-odds .sdm file over a cell box: the float cells and the `known` mask, 0 where no patch is"""
    prob, known = np.zeros((h, w), np.float32), np.zeros((h, w), np.uint8)
    ci = np.arange(PATCH * PATCH)
    for pid, (cells, mask) in f["patches"].items():
        px, py = pid // UC, pid % UC
        c = np.frombuffer(cells.tobytes(), np.float32)
        k = ((mask[ci >> 6] >> (ci & 63).astype(np.uint64)) & 1).astype(np.uint8)
        ys, xs = py * PATCH + (ci >> 5) - y0, px * PATCH + (ci & 31) - x0
        prob[ys, xs], known[ys, xs] = c, k
    return prob, known


class _Reader:
    """the readers of one device map pair: a Slam2D / LidarOdometry2D, or particle `i` of a PFSlam2D"""

    def __init__(self, g, i=None):
        self.g, self.a = g, (() if i is None else (i,))

    def window(self):
        return self.g.window()

    def __getattr__(self, name):
        f = getattr(self.g, name)
        return lambda *args: f(*self.a, *args)


def _oracle_maps(po, prefix, o, *args, okind="freq", export_occ=None):
    return dict(dm=po.map_handle(prefix + "dm", o, *args), occ=po.map_handle(prefix + "occ", o, *args), okind=okind, owner=o,
                export_occ=export_occ)


def check_readers(g, oracle_maps, window, seed=0, parked=True):
    """compares every reader of device map pair `g` (a _Reader) with the oracle's maps at this moment; `window` is g's window().
    Asserts that the probe is not vacuous: patches are parked, a stated share of the samples reaches them, some samples lie in patches
    that exist nowhere, and free, occupied and unknown cells all occur in the parked patches.  parked=False: a map that holds no
    parked patch by design (LidarOdometry2D), for which the same readers are compared after the window has moved."""
    import oracle.pyoracle as po
    from iris_lama_b200 import api
    om = oracle_maps
    assert (window["parked"] > 0) == parked, window
    rng = np.random.default_rng(seed)
    tmp = tempfile.TemporaryDirectory()
    files = {}
    for name, okind in (("occ", om["okind"]), ("dm", "ddm")):     # the oracle's maps as files: their patch sets
        assert po.map_write(okind, om[name], f"{tmp.name}/o_{name}.sdm")
        files[name] = sdm.read_sdm(f"{tmp.name}/o_{name}.sdm")
    bx, by, dim = window["base"][0], window["base"][1], window["dim"]

    def outside(px, py):
        return (px < bx) | (px >= bx + dim) | (py < by) | (py >= by + dim)

    dm_px, dm_py = _patches(files["dm"])
    occ_px, occ_py = _patches(files["occ"])
    parked_dm = (dm_px * UC + dm_py)[outside(dm_px, dm_py)]
    parked_occ = (occ_px * UC + occ_py)[outside(occ_px, occ_py)]
    assert (len(parked_dm) > 0 and len(parked_occ) > 0) == parked, (len(parked_dm), len(parked_occ))

    # ---- distance(): bit-equal to the oracle, and to a float64 bilinear reference within 1e-12 m
    pts = _probe_points(window, dm_px, dm_py, parked_dm, rng)
    dg, gg = g.distance(pts)
    dr, gr = po.DDM(handle=om["dm"].value, owner=om["owner"]).distance(pts)
    assert (dg == dr).all() and (gg == gr).all(), int((dg != dr).sum())
    lo = np.array([dm_px.min(), dm_py.min()]) * PATCH - 2 * PATCH
    hi = (np.array([dm_px.max(), dm_py.max()]) + 1) * PATCH + 2 * PATCH
    dn, gn, stencil, dmax = _bilinear_reference(po, om["dm"], pts, lo, hi)
    assert np.abs(dg - dn).max() < 1e-12 and np.abs(gg - gn).max() < 1e-9
    assert (dg[-len(FAR):] == dmax).all() and (gg[-len(FAR):] == 0).all()
    # the stencils that reach a parked patch: a stated share, some with corners in the window too; and some where no patch exists
    corners = [(stencil[:, 0] + i, stencil[:, 1] + j) for i in (0, 1) for j in (0, 1)]
    corner_ids = np.stack([_pid(x, y) for x, y in corners])
    in_window = np.stack([~outside(x >> 5, y >> 5) for x, y in corners]).any(axis=0)
    in_parked = np.isin(corner_ids, parked_dm).any(axis=0)
    assert (~np.isin(corner_ids, dm_px * UC + dm_py)).all(axis=0).any()
    if parked:
        assert in_parked.mean() >= PARKED_SHARE, in_parked.mean()
        assert (in_parked & in_window).any()

    # ---- occupancyQuery(): the cells of the points, and the rows and columns on both sides of the window's edges
    cells = [api.w2m(RES, pts[:-len(FAR)])]
    for axis, edges in ((0, (bx * PATCH, (bx + dim) * PATCH)), (1, (by * PATCH, (by + dim) * PATCH))):
        along = np.arange(lo[1 - axis] + PATCH, hi[1 - axis] - PATCH)
        for e in (edges[0] - 1, edges[0], edges[1] - 1, edges[1]):
            c = np.empty((len(along), 2), np.uint32)
            c[:, axis], c[:, 1 - axis] = e, along
            cells.append(c)
    cells = np.concatenate(cells)
    pg, fg = g.occupancyQuery(cells)
    pr, fr = po.occ_query(om["okind"], om["occ"], cells)
    assert (fg == fr).all() and (pg == pr).all(), (int((fg != fr).sum()), int((pg != pr).sum()))
    cp = np.isin(_pid(cells[:, 0], cells[:, 1]), parked_occ)
    if parked:
        assert cp.mean() >= CELL_SHARE, cp.mean()
        assert (fr[cp] & 1).any() and (fr[cp] & 2).any() and (fr[cp] & 4).any()   # free, occupied and unknown cells in parked patches

    # ---- log-odds maps: the float cells and the `known` plane over the occupancy map's bounds
    if om["okind"] == "prob":
        x0, y0 = int(occ_px.min()) * PATCH, int(occ_py.min()) * PATCH
        w, h = (int(occ_px.max()) + 1) * PATCH - x0, (int(occ_py.max()) + 1) * PATCH - y0
        eg = g.exportLogOdds(x0, y0, w, h)
        if om["export_occ"] is not None:
            eo = om["export_occ"](x0, y0, w, h)
            prob, known = eo["prob"], eo["known"]
        else:
            prob, known = _logodds_from_file(files["occ"], x0, y0, w, h)
        assert (eg["prob"].view(np.uint32) == prob.view(np.uint32)).all() and (eg["known"] == known).all()
        if parked:
            inp = np.isin(_pid(*np.meshgrid(np.arange(x0, x0 + w), np.arange(y0, y0 + h))), parked_occ)
            assert known[inp].any() and not known[inp].all()

    # ---- .sdm files (header, parameters, patch set, cells and masks) and images
    for kind, name, okind in ((0, "occ", om["okind"]), (1, "dm", "ddm")):
        g.writeMap(kind, f"{tmp.name}/g_{name}.sdm")
        _same_files(f"{tmp.name}/g_{name}.sdm", f"{tmp.name}/o_{name}.sdm")
        assert (g.exportImage(kind) == po.map_image(okind, om[name])).all(), name
    tmp.cleanup()


class _Moments:
    """the probe moments of an out-and-back run: on the way out once patches have been parked for `after` scans, on the first scan after
    the turn, and on the way back once parked patches have been restored for `after` scans"""

    def __init__(self, n_out, after=10):
        self.n_out, self.after = n_out, after
        self.back_from = n_out + 8                 # _out_and_back turns on the spot in 8 scans
        self.parked_since = self.restored_since = None
        self.restored_at_turn = None
        self.done = []

    def due(self, t, w):
        name = None
        if t < self.n_out:
            if self.parked_since is None and w["parked"] > 0:
                self.parked_since = t
            if "out" not in self.done and self.parked_since is not None and t == self.parked_since + self.after:
                name = "out"
        elif t == self.back_from:
            self.restored_at_turn = w["restored"]
            name = "turn"
        elif t > self.back_from:
            if self.restored_since is None and w["restored"] > self.restored_at_turn:
                self.restored_since = t
            if "back" not in self.done and self.restored_since is not None and t == self.restored_since + self.after:
                name = "back"
        if name:
            self.done.append(name)
        return name


def _slam_counters(g, o):
    c, _ = g.counters()
    co = o.counters()
    co = co[0] if isinstance(co, tuple) else co
    keys = ("evals", "ray_cells", "dm_pops", "gn_iters")
    return tuple(c[k] for k in keys), tuple(co[k] for k in keys)


def _check_bounds(g, o):
    for kind, (n, mn, mx) in ((0, o.occ_bounds()), (1, o.dm_bounds())):
        b = g.mapBounds(kind)
        assert (b[1] == mn).all() and (b[2] == mx).all(), kind
        if kind == 0:
            assert b[0] == n


def _check_correlation_with_parked_patches(gpu_api, po, g, o, truth, scans, t):
    """k_match while patches are parked: a candidate scan inside the window correlates as in the oracle; one that reaches parked
    ground raises LAMA_ERR_WINDOW (-4), which is sticky: the maps still read as before, and every later update fails the same way"""
    win = g.window()
    assert win["parked"] > 0
    bx, by, dim = win["base"][0], win["base"][1], win["dim"]
    od = po.DDM(handle=po.map_handle("slam_dm", o).value, owner=o)
    scan, ref = scans[t], truth[t] + np.array([0.02, 0.01, -0.01])
    for dpose in ([0.05, -0.04, 0.02], [0.3, 0.15, -0.05]):
        cand = truth[t] + np.array(dpose)
        c, s = np.cos(cand[2]), np.sin(cand[2])
        world = np.c_[cand[0] + c * scan[:, 0] - s * scan[:, 1], cand[1] + s * scan[:, 0] + c * scan[:, 1], np.zeros(len(scan))]
        cp = gpu_api.w2m(RES, world).astype(np.int64) >> 5
        assert (cp[:, 0] > bx).all() and (cp[:, 0] < bx + dim - 1).all() and (cp[:, 1] > by).all() and (cp[:, 1] < by + dim - 1).all()
        bg, eg = g.correlateCandidateScan(scan, ref, cand)
        bo, eo = od.correlate_candidate_scan(scan, ref, cand)
        assert np.abs(bg - bo).max() < POSE_TOL and abs(eg - eo) < 1e-9, dpose
    # a candidate at the far end of the corridor, wholly over parked patches
    far = int(np.argmax(truth[:, 0]))
    pts_before = g.distance(np.c_[truth[:50:5, :2], np.zeros(10)])
    with pytest.raises(gpu_api.LamaError) as e:
        g.correlateCandidateScan(scans[far], truth[far], truth[far] + np.array([0.05, -0.04, 0.02]))
    assert e.value.code == -4, e.value
    assert g.window() == win
    dg, gg = g.distance(np.c_[truth[:50:5, :2], np.zeros(10)])      # the maps are untouched and still readable
    assert (dg == pts_before[0]).all() and (gg == pts_before[1]).all()
    for k in (1, 2):
        with pytest.raises(gpu_api.LamaError) as e:
            g.update(scans[t - k], truth[t - k] + np.array([0.0, 0.0, 0.5 * k]))
        assert e.value.code == -4, (k, e.value)


@pytest.mark.parametrize("occupancy", [0, 1])
def test_slam2d_readers_over_parked_patches(gpu_api, po, synth, tmp_path, occupancy):
    truth, odom, scans = _out_and_back(synth)
    n_out = int(np.argmax(truth[:, 2] > 0))
    kw = dict(trans_thresh=0.05, rot_thresh=0.05)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(occupancy=occupancy, dir_dim=16, **kw))
    o = (po.Slam2DProb if occupancy else po.Slam2D)(po.SlamOptions.defaults(**kw))
    g.setPose(*truth[0]); o.set_pose(*truth[0])
    om = _oracle_maps(po, "slamp_" if occupancy else "slam_", o, okind="prob" if occupancy else "freq",
                      export_occ=o.export_occ if occupancy else None)
    moments, resumed = _Moments(n_out), None
    for t in range(len(scans)):
        r = o.update(scans[t], odom[t])
        assert g.update(scans[t], odom[t]) == r, t
        assert _close(g.state(), o.state()), t
        cg, co = _slam_counters(g, o)
        assert cg == co, t
        if resumed is not None:
            assert resumed.update(scans[t], odom[t]) == r and (resumed.state() == g.state()).all(), t
            assert resumed.counters()[0] == g.counters()[0], t
        m = moments.due(t, g.window())
        if m:
            check_readers(_Reader(g), om, g.window(), seed=t)
            _check_bounds(g, o)
        if m == "back":   # a checkpoint with parked entries (three kinds per map with log-odds cells)
            a, b = tmp_path / "a.ckpt", tmp_path / "b.ckpt"
            g.saveState(a)
            resumed = gpu_api.Slam2D.loadState(a)
            resumed.saveState(b)
            assert a.read_bytes() == b.read_bytes()
            rw, gw = resumed.window(), g.window()         # a loaded handle counts its own shifts and restores
            assert (rw["base"], rw["dim"], rw["parked"]) == (gw["base"], gw["dim"], gw["parked"])
            check_readers(_Reader(resumed), om, resumed.window(), seed=t)
    assert moments.done == ["out", "turn", "back"], moments.done
    w = g.window()
    assert w["shifts"] >= 3 and w["restored"] > 0 and w["parked"] > 0, w
    for h in (g, resumed):
        check_readers(_Reader(h), om, h.window(), seed=1)
    _check_bounds(g, o)
    if occupancy == 0:
        _check_correlation_with_parked_patches(gpu_api, po, g, o, truth, scans, len(scans) - 1)


@pytest.mark.parametrize("gain", [0.02, 0.1])
def test_pfslam2d_particle_readers_over_parked_patches(gpu_api, po, synth, gain):
    """gain 0.02: sharp weights, the filter resamples every few scans (some 65 times), so a patch is no longer owned by one particle when it
    is parked.  gain 0.1: eight resamplings, far enough apart that patches written since the last one are parked while a particle
    still owns them (kDirOwn), and the next resampling shares those entries between the copies of that particle: their shared slots
    must go through copy-on-write when the robot comes back and the restored patches are written."""
    truth, odom, scans = _out_and_back(synth, step=0.3)
    n_out = int(np.argmax(truth[:, 2] > 0))
    P = 16
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, seed=5, meas_sigma_gain=gain)
    g = gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(P, dir_dim=16, **kw))
    o = po.PFSlam2D(po.PFOptions.defaults(P, **kw))
    g.setPrior(*truth[0]); o.set_prior(*truth[0])
    moments, copied_from, probed = _Moments(n_out), None, []
    for t in range(len(scans)):
        r = o.update(scans[t], odom[t])
        assert g.update(scans[t], odom[t]) == r, t
        so, _ = o.particles()
        sg, _ = g.getParticles()
        assert _close(sg, so), t
        lo = o.last_resample()
        assert (np.asarray(g.lastResample()) == lo).all(), t
        w = g.window()
        if g.counters()[0]["resampled"] and w["parked"] > 0:
            copied_from = np.asarray(lo)                 # this resampling copied parked lists (k_copy_parked)
        m = moments.due(t, w)
        if m:
            ids = [0, g.getBestParticleIdx()]
            if copied_from is not None:
                moved = np.flatnonzero(copied_from != np.arange(P))
                assert len(moved), copied_from
                ids.append(int(moved[0]))
            for i in dict.fromkeys(ids):
                check_readers(_Reader(g, i), _oracle_maps(po, "pf_", o, i), w, seed=t + i)
            probed.append((m, copied_from is not None))
    assert moments.done == ["out", "turn", "back"], moments.done
    assert probed[1:] == [("turn", True), ("back", True)], probed    # from the turn on, a resampled copy of parked lists is probed too
    w = g.window()
    assert w["shifts"] >= 3 and w["restored"] > 0 and w["parked"] > 0, w
    for i in range(P):
        check_readers(_Reader(g, i), _oracle_maps(po, "pf_", o, i), w, seed=i)




def test_slam2d_logodds_transient_map_prunes_parked_patches(gpu_api, po, synth):
    """log-odds cells, truncated rays and a transient map with 30 m beams: the map's box (pose +- twice the scan's extent) reaches past
    a window centred on the robot, so parked patches of all three kinds (occupancy, distance and the ray cast's scratch counters)
    survive prunes, and later prunes delete them in place"""
    truth, odom, scans = _out_and_back(synth, length=150.0, step=0.6, r_max=30.0)
    n_out = int(np.argmax(truth[:, 2] > 0))
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, transient_map=1, truncated_ray=6.0)
    g = gpu_api.Slam2D(gpu_api.Slam2D.Options(occupancy=1, **kw))
    o = po.Slam2DProb(po.SlamOptions.defaults(**kw))
    g.setPose(*truth[0]); o.set_pose(*truth[0])
    om = _oracle_maps(po, "slamp_", o, okind="prob", export_occ=o.export_occ)
    po.lib().orc_slamp_removed_patches.restype = po.C.c_uint64
    probes, shrunk, prev = [], 0, 0
    for t in range(n_out):
        assert g.update(scans[t], odom[t]) == o.update(scans[t], odom[t])
        assert _close(g.state(), o.state()), t
        cg, co = _slam_counters(g, o)
        assert cg == co, t
        assert g.mapStats()[1] == po.lib().orc_slamp_removed_patches(o.h), t
        w = g.window()
        if 0 < w["parked"] < prev:
            shrunk += 1                                   # a prune deleted parked entries and kept others
            if len(probes) < 3:
                check_readers(_Reader(g), om, w, seed=t)
                probes.append(t)
        prev = w["parked"]
    assert shrunk >= 2 and len(probes) == min(3, shrunk), (shrunk, probes)
    _check_bounds(g, o)


def test_lidar_odometry_30m_beams_hold_no_parked_patch(gpu_api, po, synth):
    """LidarOdometry2D with 30 m beams along 150 m (log-odds cells, 1 m rays, a transient map).  Its transient box (pose +- the scan's
    extent + two reaches) lies inside the guarded box the window is centred to hold, so after every update the map has no patch outside
    the window: nothing stays parked.  Pinned, with every reader compared against the oracle after the window has moved."""
    truth, odom, scans = _out_and_back(synth, length=150.0, step=0.3, r_max=30.0, n_beams=720)
    n_out = int(np.argmax(truth[:, 2] > 0))
    g, o = gpu_api.LidarOdometry2D(), po.LidarOdometry2D()
    for t in range(n_out):
        assert g.update(scans[t]) == o.update(scans[t])
        assert _close(g.state(), o.state()), t
        c = o.counters()
        assert g.mapStats() == (c["map_updates"], c["removed_patches"]), t
        assert g.window()["parked"] == 0, t
    w = g.window()
    assert w["shifts"] >= 3 and c["removed_patches"] > 0 and g.getPose()[0] > 140.0, (w, c, g.getPose())
    check_readers(_Reader(g), _oracle_maps(po, "lo_", o, okind="prob"), w, parked=False)
