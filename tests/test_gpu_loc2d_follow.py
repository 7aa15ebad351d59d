"""Localisation in maps larger than the device window: a following DynamicDistanceMap (lama_dm_set_follow) and Loc2D on it, driven
along corridors longer than the window.  Checked against the oracle, whose maps have no edge, and against the same run in a fixed window
large enough never to move: the shifts, the parked patches and the whole-map global localisation must not show in any result."""
import numpy as np
import pytest

from test_gpu_window_follow import _close, _out_and_back
from test_sdm_io import _same_files

pytestmark = pytest.mark.gpu

O = 1321122 * 32
FIELDS = ("sqdist", "valid", "ox", "oy", "queued", "known")
KW = dict(trans_thresh=0.2, rot_thresh=0.2, cov_blend=0.5)
DEV = dict(max_beams=512)   # a 128-patch window fits the shared-memory budget


def _cells(segments):
    cells = set()
    for x1, y1, x2, y2 in segments:
        n = int(max(abs(x2 - x1), abs(y2 - y1)) / 0.05) + 1
        for k in range(n + 1):
            cells.add((int((x1 + (x2 - x1) * k / n) * 20 + O + 0.5), int((y1 + (y2 - y1) * k / n) * 20 + O + 0.5)))
    return np.array(sorted(cells), np.uint32)


def _free(length):
    """every other cell inside the corridor of make_corridor(length): x in (-2, length - 2), |y| < 1"""
    xs = np.arange(int(-1.9 * 20), int((length - 2.1) * 20), 2)
    ys = np.arange(int(-0.9 * 20), int(0.9 * 20) + 1, 2)
    return np.array([(x + O, y + O) for x in xs for y in ys], np.uint32)


def _oracle_file(po, cells, path, l2_max=1.0):
    od = po.DDM(0.05, 32, l2_max)
    od.add(cells)
    od.update()
    assert po.map_write("ddm", od, path)
    return od


def _export_equal(g, od):
    n, mn, mx = od.bounds()
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g.export(int(mn[0]), int(mn[1]), w, h), od.export(mn[0], mn[1], w, h)
    for k in FIELDS:
        assert (a[k] == b[k]).all(), f"{k}: {int((a[k] != b[k]).sum())} cells differ"
    assert g.bounds()[0] == n


def _loc(gpu_api, po, path, cells, dir_dim, follow, **kw):
    gl = gpu_api.Loc2D(gpu_api.Loc2D.Options(dir_dim=dir_dim, **DEV, **KW, **kw))
    if follow:
        gl.distance_map.setFollow(True)
    gl.distance_map.read(path)
    return gl


def _step(hs, ol, scan, odom, t, force):
    """one update of every device handle and the oracle: the device runs bit-equal, each within tolerance of the oracle -- the pose and
    RMSE per metre from the origin, the covariance within 1e-8 of its largest entry (its cross terms are small in a corridor)"""
    r = ol.update(scan, odom, force=force)
    sc, cov, rmse, _ = ol.get()
    for g in hs:
        assert g.update(scan, odom, force_update=force) == r, t
    for g in hs[1:]:
        assert (g.state() == hs[0].state()).all() and g.getRMSE() == hs[0].getRMSE() and (g.getCovar() == hs[0].getCovar()).all(), t
    for g in hs:
        assert _close(g.state(), sc), (t, g.state(), sc)
        assert abs(g.getRMSE() - rmse) < 1e-11 * max(1.0, float(np.abs(sc[2:]).max())), t
        assert np.abs(g.getCovar() - cov).max() <= 1e-8 * np.abs(cov).max(), (t, g.getCovar(), cov)
        assert g.globalLocalizationActive() == ol.gloc_active(), t


@pytest.fixture(scope="module")
def corridor(synth, po, tmp_path_factory):
    truth, odom, scans = _out_and_back(synth)
    cells = _cells(synth.make_corridor(length=84.0))
    path = tmp_path_factory.mktemp("loc2d_follow") / "corridor.sdm"
    od = _oracle_file(po, cells, path)
    return dict(truth=truth, odom=odom, scans=scans, cells=cells, path=path, od=od)


def test_file_round_trip(gpu_api, po, corridor, tmp_path):
    path = corridor["path"]
    g16 = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, follow=True, dir_dim=16, **DEV)
    g128 = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, dir_dim=128, **DEV)
    g16.read(path)
    g128.read(path)
    w = g16.window()
    assert w["parked"] > 0 and w["base"] == gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, dir_dim=16).window()["base"], w   # back where it was
    for name, g in (("g16", g16), ("g128", g128)):
        g.write(tmp_path / f"{name}.sdm")
        _same_files(str(path), str(tmp_path / f"{name}.sdm"))
        _export_equal(g, corridor["od"])
    fixed = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, dir_dim=16)
    with pytest.raises(gpu_api.LamaError) as e:
        fixed.read(path)
    assert e.value.code == -4


def test_tracking_out_and_back(gpu_api, po, corridor):
    c = corridor
    g16 = _loc(gpu_api, po, c["path"], c["cells"], 16, True)
    g128 = _loc(gpu_api, po, c["path"], c["cells"], 128, False)
    ol = po.Loc2D(po.LocOptions.defaults(**KW))
    od = ol.dm(); od.add(c["cells"]); od.update()
    for h in (g16, g128):
        h.setPose(*c["truth"][0])
    ol.set_pose(*c["truth"][0])
    for t in range(len(c["scans"])):
        _step([g16, g128], ol, c["scans"][t], c["odom"][t], t, t == 0)
    w16, w128 = g16.distance_map.window(), g128.distance_map.window()
    assert w16["shifts"] >= 3 and w16["restored"] > 0 and w16["parked"] > 0, w16
    assert w128["shifts"] == 0 and w128["parked"] == 0, w128


def test_global_localization_over_the_whole_map(gpu_api, po, corridor):
    c = corridor
    kw = dict(gloc_particles=3000, timing=1)
    g16 = _loc(gpu_api, po, c["path"], c["cells"], 16, True, **kw)
    g128 = _loc(gpu_api, po, c["path"], c["cells"], 128, False, **kw)
    ol = po.Loc2D(po.LocOptions.defaults(gloc_particles=3000, **KW))
    od = ol.dm(); od.add(c["cells"]); od.update()
    free = _free(84.0)
    for h in (g16, g128):
        h.occupancySet(free, -1); h.occupancySet(c["cells"], 1); h.setSeed(91)
    ol.occ_set(free, -1); ol.occ_set(c["cells"], 1); ol.set_seed(91)
    t0 = 100   # start 25 m down the corridor, the pose set 40 m away from it
    x, y, r = c["truth"][t0]
    for h in (g16, g128):
        h.setPose(x - 40.0, y, r + 1.0); h.triggerGlobalLocalization()
    ol.set_pose(x - 40.0, y, r + 1.0); ol.trigger_global_localization()
    gloc_steps = 0
    for t in range(t0, t0 + 40):
        active = ol.gloc_active()
        before = [h.distance_map.kernelTimes()[1]["match"] for h in (g16, g128)]
        parked = g16.distance_map.window()["parked"]
        _step([g16, g128], ol, c["scans"][t], c["odom"][t], t, t == t0)
        after = [h.distance_map.kernelTimes()[1]["match"] for h in (g16, g128)]
        assert after[0] - before[0] == after[1] - before[1], t   # the whole-map scoring is one launch, as the in-window one
        if active and after[1] - before[1] >= 2 + (t == t0):
            gloc_steps += 1
            assert parked > 0, t                                     # so the 16-patch run scored its candidates over parked patches
    assert gloc_steps >= 1
    assert not g16.globalLocalizationActive()


def test_obstacles_on_a_following_map(gpu_api, po, corridor, tmp_path):
    path = corridor["path"]
    g16 = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, follow=True, dir_dim=16, **DEV)
    g128 = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, dir_dim=128, **DEV)
    for g in (g16, g128):
        g.read(path)
    rng = np.random.default_rng(5)

    def blob(x_m, n):   # n distinct cells inside the corridor within 4 m of x_m, sorted
        x0 = int((x_m - 4) * 20) + O
        k = np.sort(rng.choice(160 * 31, n, replace=False))
        return np.stack([x0 + k // 31, O - 15 + k % 31], 1).astype(np.uint32)

    far = blob(60.0, 2600)                  # over parked ground, more than one chunk
    near = blob(5.0, 900)
    batches = [("add", far), ("add", near), ("remove", far[::3]), ("add", np.concatenate([blob(45.0, 2048), blob(70.0, 600)])),
               ("remove", near[::2])]
    for k, (op, cells) in enumerate(batches):
        for g in (g16, g128):
            (g.addObstacle if op == "add" else g.removeObstacle)(cells)
        assert g16.update() == g128.update(), k
    assert g16.window()["shifts"] >= 2 and g16.window()["parked"] > 0
    n, mn, mx = g128.bounds()
    assert g16.bounds()[0] == n
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = g16.export(int(mn[0]), int(mn[1]), w, h), g128.export(int(mn[0]), int(mn[1]), w, h)
    for key in FIELDS:
        assert (a[key] == b[key]).all(), key
    before, after = tmp_path / "before.sdm", tmp_path / "after.sdm"
    g16.write(before)
    wide = np.array([(O + 200, O), (O + 200 + 16 * 32, O)], np.uint32)   # one chunk spanning more than 16 patches
    g16.addObstacle(wide)
    with pytest.raises(gpu_api.LamaError) as e:
        g16.update()
    assert e.value.code == -4
    g16.write(after)
    assert before.read_bytes() == after.read_bytes()


def test_pool_grows_or_refuses(gpu_api, po, tmp_path):
    # a 70 m x 70 m grid of obstacles every 1.6 m: more patches than the automatic pool (1 792 slots) holds
    g = np.arange(-700, 700, 32)
    cells = np.array([(x + O, y + O) for x in g for y in g], np.uint32)
    path = tmp_path / "grid.sdm"
    od = _oracle_file(po, cells, path)
    n = od.bounds()[0]
    assert n > 1792
    small = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, follow=True, dir_dim=16, pool_slots=1000)
    with pytest.raises(gpu_api.LamaError) as e:
        small.read(path)
    assert e.value.code == -5
    assert small.bounds()[0] == 0 and small.window()["shifts"] == 0   # nothing was written
    rd = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, follow=True, dir_dim=16)
    assert rd.pool()[0] == 1792
    rd.read(path)
    assert rd.pool()[0] > 1792 and rd.pool()[1] == n, rd.pool()
    rd.write(tmp_path / "rd.sdm")
    _same_files(str(path), str(tmp_path / "rd.sdm"))
    # the same grid through update(), in bands of rows (one brushfire over all of it would overflow the brushfire heap); the grid fits
    # this window, so the pool grows before the bands that need it
    up = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, follow=True, dir_dim=64)
    ref = gpu_api.DynamicDistanceMap(0.05, l2_max=1.0, dir_dim=128, pool_slots=8192, **DEV)
    for band in np.array_split(np.arange(len(g)), 8):
        rows = cells[np.isin(cells[:, 1], g[band] + O)]
        for m in (up, ref):
            m.addObstacle(rows)
        assert up.update() == ref.update()
    assert up.pool()[0] > 1792 and up.pool()[1] == ref.pool()[1] and up.bounds()[0] == ref.bounds()[0], (up.pool(), ref.pool())
    mn, mx = od.bounds()[1:]
    w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
    a, b = up.export(int(mn[0]), int(mn[1]), w, h), ref.export(int(mn[0]), int(mn[1]), w, h)
    for key in FIELDS:
        assert (a[key] == b[key]).all(), key


def test_corridor_longer_than_the_largest_window(gpu_api, po, synth, tmp_path):
    length = 300.0
    truth, odom, scans = _out_and_back(synth, length=length, step=0.5)
    half = len(truth) // 2                       # the way out: past 204 m, the width of a 128-patch window
    cells = _cells(synth.make_corridor(length=length))
    path = tmp_path / "long.sdm"
    od = _oracle_file(po, cells, path)
    gl = gpu_api.Loc2D(gpu_api.Loc2D.Options(dir_dim=128, gloc_particles=3000, **DEV, **KW))
    gl.distance_map.setFollow(True)
    gl.distance_map.read(path)
    gl.distance_map.write(tmp_path / "g.sdm")
    _same_files(str(path), str(tmp_path / "g.sdm"))
    _export_equal(gl.distance_map, od)
    ol = po.Loc2D(po.LocOptions.defaults(gloc_particles=3000, **KW))
    o = ol.dm(); o.add(cells); o.update()
    gl.setPose(*truth[0]); ol.set_pose(*truth[0])
    for t in range(half):
        _step([gl], ol, scans[t], odom[t], t, t == 0)
    assert truth[half - 1][0] > 204.8 and gl.distance_map.window()["parked"] > 0
    free = _free(length)
    gl.occupancySet(free, -1); gl.occupancySet(cells, 1); gl.setSeed(5)
    ol.occ_set(free, -1); ol.occ_set(cells, 1); ol.set_seed(5)
    x, y, r = truth[half - 1]
    gl.setPose(x - 150.0, y, r); ol.set_pose(x - 150.0, y, r)
    gl.triggerGlobalLocalization(); ol.trigger_global_localization()
    for t in range(half - 1, half + 11):
        _step([gl], ol, scans[t], odom[t], t, t == half - 1)
