"""The 2-D maps' moving window on the device: PFSlam2D, Slam2D and LidarOdometry2D driven further than their directory window, which
follows the robot (Engine::shift_window) and parks the patches it leaves.  Checked against the oracle, whose maps have no edge, and
against the same run in a window large enough never to move: the shifts must not show in any result."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-9   # per metre of distance from the origin: the runs reach 230 m


def _close(a, b):
    return np.abs(a - b).max() < POSE_TOL * max(1.0, float(np.abs(b).max()))


def _out_and_back(synth, length=84.0, step=0.25, r_max=8.0, n_beams=360, laps=1):
    """a corridor of `length` m driven to its far end and back (`laps` times), beams shorter than r_max"""
    segs = synth.make_corridor(length=length)
    xs = np.arange(0.0, length - 6.0, step)
    turn = np.linspace(0.0, np.pi, 10)[1:-1]
    path = []
    for _ in range(laps):
        path += [(x, 0.05 * np.sin(0.7 * x), 0.0) for x in xs] + [(xs[-1], 0.0, a) for a in turn]
        path += [(x, 0.05 * np.sin(0.7 * x), np.pi) for x in xs[::-1]] + [(xs[0], 0.0, np.pi - a) for a in turn]
    truth = np.array(path)
    angles = synth.beam_angles(n_beams, 360.0)
    rng_r, rng_o = np.random.default_rng(11), np.random.default_rng(12)
    scans, odom = [], np.zeros_like(truth)
    cur = tuple(truth[0])
    for t in range(len(truth)):
        r = synth.cast(segs, truth[t], angles, 30.0) + rng_r.normal(0.0, 0.01, n_beams)
        p = synth.scan_points(r, angles)
        scans.append(np.ascontiguousarray(p[np.hypot(p[:, 0], p[:, 1]) < r_max]))
        if t == 0:
            odom[0] = truth[0]
        else:
            d = synth._between(tuple(truth[t - 1]), tuple(truth[t]))
            cur = synth._compose(cur, (d[0] + rng_o.normal(0, 0.01), d[1] + rng_o.normal(0, 0.01), d[2] + rng_o.normal(0, 0.005)))
            odom[t] = cur
    return truth, odom, scans


def _assert_maps_equal(a_dm, b_dm, a_occ, b_occ):
    for k in ("sqdist", "valid", "ox", "oy", "queued", "known"):
        assert (a_dm[k] == b_dm[k]).all(), f"{k}: {int((a_dm[k] != b_dm[k]).sum())} cells differ"
    for k in ("occupied", "visited", "known"):
        assert (a_occ[k] == b_occ[k]).all(), k


def test_slam2d_follows_the_robot(gpu_api, po, synth, tmp_path):
    truth, odom, scans = _out_and_back(synth)
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, max_beams=512)   # max_beams 512: a 128-patch window fits the shared-memory budget
    g16 = gpu_api.Slam2D(gpu_api.Slam2D.Options(dir_dim=16, **kw))
    g128 = gpu_api.Slam2D(gpu_api.Slam2D.Options(dir_dim=128, **kw))
    o = po.Slam2D(po.SlamOptions.defaults(trans_thresh=0.05, rot_thresh=0.05))
    for h in (g16, g128):
        h.setPose(*truth[0])
    o.set_pose(*truth[0])
    resumed, t_save = None, len(scans) // 2 + 40   # on the way back, over parked patches
    for t in range(len(scans)):
        r = o.update(scans[t], odom[t])
        assert g16.update(scans[t], odom[t]) == r and g128.update(scans[t], odom[t]) == r, t
        assert _close(g16.state(), o.state()), t
        assert (g16.state() == g128.state()).all(), t
        c16, _ = g16.counters(); c128, _ = g128.counters(); co, _ = o.counters()
        assert (c16["evals"], c16["ray_cells"], c16["dm_pops"], c16["gn_iters"]) == (co["evals"], co["ray_cells"], co["dm_pops"], co["gn_iters"]), t
        assert c16 == c128, t
        if resumed is not None:
            assert resumed.update(scans[t], odom[t]) == r and (resumed.state() == g16.state()).all() and resumed.counters()[0] == c16, t
        if t == t_save:   # a checkpoint with parked entries: loaded into a new handle, which continues bit for bit
            assert g16.window()["parked"] > 0
            a, b = tmp_path / "a.ckpt", tmp_path / "b.ckpt"
            g16.saveState(a)
            resumed = gpu_api.Slam2D.loadState(a)
            resumed.saveState(b)
            assert a.read_bytes() == b.read_bytes()                   # save -> load -> save gives the same bytes
            assert resumed.window()["parked"] == g16.window()["parked"]
    w16, w128 = g16.window(), g128.window()
    assert w16["shifts"] >= 3 and w16["restored"] > 0 and w16["parked"] > 0, w16
    assert w128["shifts"] == 0 and w128["parked"] == 0, w128
    assert g16.counters()[1] == g128.counters()[1]      # totals, detached patches included
    for kind, ob in ((1, o.dm_bounds()), (0, o.occ_bounds())):
        n, mn, mx = ob
        b16, b128 = g16.mapBounds(kind), g128.mapBounds(kind)
        assert (b16[1] == mn).all() and (b16[2] == mx).all() and (b128[1] == mn).all() and (b128[2] == mx).all()
        assert b16[0] == b128[0]
        if kind == 0:
            assert b16[0] == n
    n, mn, mx = o.dm_bounds()
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    eo_dm, eo_occ = o.export_dm(mn[0], mn[1], w, h), o.export_occ(mn[0], mn[1], w, h)
    for g in (g16, g128, resumed):
        _assert_maps_equal(g.exportDistance(int(mn[0]), int(mn[1]), w, h), eo_dm, g.exportOccupancy(int(mn[0]), int(mn[1]), w, h), eo_occ)
    for kind in (0, 1):
        a, b = str(tmp_path / f"a{kind}.sdm"), str(tmp_path / f"b{kind}.sdm")
        g16.writeMap(kind, a)
        g128.writeMap(kind, b)
        assert open(a, "rb").read() == open(b, "rb").read()


def test_pfslam2d_follows_the_robot(gpu_api, po, synth, tmp_path):
    truth, odom, scans = _out_and_back(synth, step=0.3)
    P = 16
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, seed=5, meas_sigma_gain=0.02)   # sharp weights: the filter resamples often (65 times)
    g16 = gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(P, dir_dim=16, max_beams=512, **kw))
    g128 = gpu_api.PFSlam2D(gpu_api.PFSlam2D.Options(P, dir_dim=128, max_beams=512, **kw))
    o = po.PFSlam2D(po.PFOptions.defaults(P, **kw))
    for h in (g16, g128):
        h.setPrior(*truth[0])
    o.set_prior(*truth[0])
    first_shift, resampled_after = None, 0
    resumed, t_save = None, len(scans) // 2 + 30
    for t in range(len(scans)):
        r = o.update(scans[t], odom[t])
        assert g16.update(scans[t], odom[t]) == r and g128.update(scans[t], odom[t]) == r, t
        so, _ = o.particles()
        s16, _ = g16.getParticles()
        s128, _ = g128.getParticles()
        assert _close(s16, so), t
        assert (s16 == s128).all(), t
        lo = o.last_resample()
        assert (np.asarray(g16.lastResample()) == lo).all() and (np.asarray(g128.lastResample()) == lo).all(), t
        # every counter but `detached`: two particles that write a patch they share in the same update copy it once or twice, as
        # their CTAs happen to finish -- a race the window size changes, not the shift
        c16, _ = g16.counters()
        c128 = g128.counters()[0]
        assert {k: v for k, v in c16.items() if k != "detached"} == {k: v for k, v in c128.items() if k != "detached"}, t
        if resumed is not None:
            assert resumed.update(scans[t], odom[t]) == r and (resumed.getParticles()[0] == s16).all(), t
            cr = resumed.counters()[0]
            assert (np.asarray(resumed.lastResample()) == lo).all() and all(cr[k] == c16[k] for k in c16 if k != "detached"), t
        if t == t_save:   # a checkpoint with parked entries continues bit for bit; save -> load -> save gives the same bytes
            assert g16.window()["parked"] > 0
            a, b = tmp_path / "a.ckpt", tmp_path / "b.ckpt"
            g16.saveState(a)
            resumed = gpu_api.PFSlam2D.loadState(a)
            resumed.saveState(b)
            assert a.read_bytes() == b.read_bytes()
        if first_shift is None and g16.window()["shifts"]:
            first_shift = t
        elif first_shift is not None and c16["resampled"]:
            resampled_after += 1
    w16 = g16.window()
    assert w16["shifts"] >= 3 and w16["restored"] > 0 and w16["parked"] > 0, w16
    assert g128.window()["shifts"] == 0
    assert resampled_after >= 3, resampled_after
    for i in (0, 5, P - 1):
        n, mn, mx = o.dm_bounds(i)
        w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
        _assert_maps_equal(g16.exportDistance(i, int(mn[0]), int(mn[1]), w, h), o.export_dm(i, mn[0], mn[1], w, h),
                           g16.exportOccupancy(i, int(mn[0]), int(mn[1]), w, h), o.export_occ(i, mn[0], mn[1], w, h))
        n, mn, mx = o.occ_bounds(i)
        b = g16.mapBounds(i, 0)
        assert b[0] == n and (b[1] == mn).all() and (b[2] == mx).all()
    # memory usage, parked patches included, as without a shift (against the oracle only the occupancy part is exact: the distance
    # maps' share is an upper estimate, Engine::memory_usage)
    m16, m128, mo = tuple(g16.getMemoryUsage()), tuple(g128.getMemoryUsage()), o.memory_usage()
    assert m16 == m128 and m16[1] == mo[1]
    assert tuple(resumed.getMemoryUsage()) == m16
    # migration blobs do not carry parked entries: refused
    with pytest.raises(gpu_api.LamaError) as e:
        g16.packParticle(0)
    assert e.value.code == -7 and "parked" in str(e.value)


def test_lidar_odometry_beyond_the_largest_window(gpu_api, po, synth):
    """a 230 m corridor: further than a 128-patch window (204.8 m) reaches; the transient map deletes what it parks"""
    truth, odom, scans = _out_and_back(synth, length=230.0, step=0.3, r_max=3.0, n_beams=720)
    n_out = int(np.argmax(truth[:, 2] > 0))   # the far end
    g, o = gpu_api.LidarOdometry2D(), po.LidarOdometry2D()
    for t in range(n_out):
        assert g.update(scans[t]) == o.update(scans[t])
        assert _close(g.state(), o.state()), t
        assert g.window()["parked"] == 0, t
    c = o.counters()
    assert g.mapStats() == (c["map_updates"], c["removed_patches"])
    assert g.window()["shifts"] >= 3 and g.getPose()[0] > 150.0


def test_slam2d_transient_map_beyond_the_largest_window(gpu_api, po, synth):
    truth, odom, scans = _out_and_back(synth, length=230.0, step=0.3, r_max=1.5, n_beams=720)
    n_out = int(np.argmax(truth[:, 2] > 0))
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, transient_map=1)
    g, o = gpu_api.Slam2D(gpu_api.Slam2D.Options(**kw)), po.Slam2D(po.SlamOptions.defaults(**kw))
    g.setPose(*truth[0]); o.set_pose(*truth[0])
    for t in range(n_out):
        assert g.update(scans[t], odom[t]) == o.update(scans[t], odom[t])
        assert _close(g.state(), o.state()), t
        assert g.window()["parked"] == 0, t
    po.lib().orc_slam_removed_patches.restype = po.C.c_uint64
    assert g.mapStats()[1] == po.lib().orc_slam_removed_patches(o.h)
    assert g.window()["shifts"] >= 2 and truth[n_out - 1, 0] > 204.8


def test_slam2d_transient_map_keeps_parked_patches_inside_its_box(gpu_api, po, synth):
    """30 m beams: the transient map's box (pose +- twice the scan's extent) reaches past a window centred on the robot, so parked
    patches survive prunes, later prunes shorten the parked lists in place, and the window keeps moving over them"""
    truth, odom, scans = _out_and_back(synth, length=150.0, step=0.6, r_max=30.0)
    n_out = int(np.argmax(truth[:, 2] > 0))
    kw = dict(trans_thresh=0.05, rot_thresh=0.05, transient_map=1)
    g, o = gpu_api.Slam2D(gpu_api.Slam2D.Options(**kw)), po.Slam2D(po.SlamOptions.defaults(**kw))
    g.setPose(*truth[0]); o.set_pose(*truth[0])
    po.lib().orc_slam_removed_patches.restype = po.C.c_uint64
    most, shifts_after = 0, 0
    for t in range(n_out):
        assert g.update(scans[t], odom[t]) == o.update(scans[t], odom[t])
        assert _close(g.state(), o.state()), t
        assert g.mapStats()[1] == po.lib().orc_slam_removed_patches(o.h), t
        w = g.window()
        if most and w["shifts"] > shifts_before:
            shifts_after += 1
        shifts_before = w["shifts"]
        most = max(most, w["parked"])
    assert most > 0 and shifts_after >= 1, (most, shifts_after)
    n, mn, mx = o.dm_bounds()
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    _assert_maps_equal(g.exportDistance(mn[0], mn[1], w, h), o.export_dm(mn[0], mn[1], w, h), g.exportOccupancy(mn[0], mn[1], w, h),
                       o.export_occ(mn[0], mn[1], w, h))
