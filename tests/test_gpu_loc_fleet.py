"""Loc2DFleet: many robots localising on one shared map.  Robot r of a fleet must give, bit for bit, what a stand-alone Loc2D with the
same options, map and seed gives when it is fed only r's calls in the same order, whatever the other robots of a call; and, like
Loc2D, stay within the oracle's tolerances (test_gpu_loc2d_follow._step)."""
import numpy as np
import pytest

from test_gpu_loc2d_follow import _cells, _free, _oracle_file
from test_gpu_window_follow import _close, _out_and_back

pytestmark = pytest.mark.gpu

KW = dict(trans_thresh=0.3, rot_thresh=0.2, cov_blend=0.5)   # 0.25 m steps: every other scan stays below the gate
WIDE = dict(dir_dim=64, center=(40.0, 0.0))                   # a fixed window over the whole 84 m corridor


@pytest.fixture(scope="module")
def corridor(synth, po, tmp_path_factory):
    data = {}
    for nb in (180, 360, 720, 1080):
        truth, odom, scans = _out_and_back(synth, n_beams=nb, r_max=30.0 if nb > 360 else 8.0)
        data[nb] = dict(truth=truth, odom=odom, scans=scans)
    cells = _cells(synth.make_corridor(length=84.0))
    path = tmp_path_factory.mktemp("loc_fleet") / "corridor.sdm"
    _oracle_file(po, cells, path)
    return dict(data=data, cells=cells, path=path)


def _mount(r):
    a = 0.01 * r
    return np.array([0.02 * r, -0.01 * r, 0.0]), np.array([0.0, 0.0, np.sin(a / 2), np.cos(a / 2)])


def _fleet(gpu_api, c, robots, follow=False, **kw):
    f = gpu_api.Loc2DFleet(gpu_api.Loc2DFleet.Options(**kw), robots)
    if follow:
        f.distance_map.setFollow(True)
    f.distance_map.read(c["path"])
    return f


def _single(gpu_api, c, follow=False, **kw):
    g = gpu_api.Loc2D(gpu_api.Loc2D.Options(**kw))
    if follow:
        g.distance_map.setFollow(True)
    g.distance_map.read(c["path"])
    return g


def _oracle(po, c, **kw):
    ol = po.Loc2D(po.LocOptions.defaults(**kw))
    od = ol.dm()
    od.add(c["cells"])
    od.update()
    return ol


def _same(f, r, g, what):
    st, cov, rmse, stats = f._get()
    assert (st[r] == g.state()).all(), (what, r, st[r], g.state())
    assert rmse[r] == g.getRMSE(), (what, r)
    assert (cov[r] == g.getCovar()).all(), (what, r)
    assert (stats[r] == g.solveStats()).all(), (what, r)
    assert f.globalLocalizationActive(r) == g.globalLocalizationActive(), (what, r)


def _near_oracle(f, r, ol, what):
    sc, cov, rmse, _ = ol.get()
    st, fc, fr, _ = f._get()
    assert _close(st[r], sc), (what, r, st[r], sc)
    assert abs(fr[r] - rmse) < 1e-11 * max(1.0, float(np.abs(sc[2:]).max())), what
    assert np.abs(fc[r] - cov).max() <= 1e-8 * np.abs(cov).max(), (what, r)
    assert f.globalLocalizationActive(r) == ol.gloc_active(), (what, r)


def _run(f, hs, ols, c, plan, mounts=None, beams=None, before_round=None):
    """plan: per round a list of (robot, scan index); robot r takes its dataset's scan and odometry at that index"""
    for i, batch in enumerate(plan):
        if before_round:
            before_round(i)
        robots = [r for r, _ in batch]
        data = [c["data"][beams[r] if beams else 360] for r in robots]
        scans = [d["scans"][t] for d, (_, t) in zip(data, batch)]
        odoms = [d["odom"][t] for d, (_, t) in zip(data, batch)]
        force = [hs[r].first for r in robots]
        kw = {}
        if mounts:
            kw = dict(origins=[mounts[r][0] for r in robots], quats=[mounts[r][1] for r in robots])
        did = f.update(robots, scans, odoms, force=force, **kw)
        for k, r in enumerate(robots):
            mk = dict(origin=mounts[r][0], quat=mounts[r][1]) if mounts else {}
            assert hs[r].update(scans[k], odoms[k], force_update=force[k], **mk) == did[k], (i, r)
            hs[r].first = False
            if ols:
                assert ols[r].update(scans[k], odoms[k], force=force[k], **mk) == did[k], (i, r)
        for r in robots:
            _same(f, r, hs[r], i)
            if ols:
                _near_oracle(f, r, ols[r], i)


def _place(f, hs, ols, starts, c, beams=None):
    for r, t in enumerate(starts):
        x, y, a = c["data"][beams[r] if beams else 360]["truth"][t]
        f.setPose(r, x, y, a)
        hs[r].setPose(x, y, a)
        hs[r].first = r == 0   # robot 0 is forced on its first scan
        if ols:
            ols[r].set_pose(x, y, a)


def test_tracking_matches_stand_alone_and_oracle(gpu_api, po, corridor):
    c = corridor
    R = 8
    beams = [180, 360, 720, 1080, 1080, 720, 360, 180]
    starts = [0, 40, 80, 120, 200, 300, 330, 420]
    f = _fleet(gpu_api, c, R, **WIDE, **KW)
    hs = [_single(gpu_api, c, **WIDE, **KW) for _ in range(R)]
    ols = [_oracle(po, c, **KW) for _ in range(R)]
    _place(f, hs, ols, starts, c, beams)
    rng = np.random.default_rng(3)
    plan = []
    for i in range(24):
        rs = [r for r in range(R) if (i + r) % 4 != 3]   # each robot skips every fourth round
        rng.shuffle(rs)
        plan.append([(r, starts[r] + i) for r in rs])
    mounts = [_mount(r) for r in range(R)]
    _run(f, hs, ols, c, plan, mounts=mounts, beams=beams)
    assert len({int(n) for n in (c["data"][b]["scans"][starts[r]].shape[0] for r, b in enumerate(beams))}) >= 4


@pytest.mark.parametrize("cov_blend", [0.0, 0.5])
def test_batch_composition_does_not_show(gpu_api, po, corridor, cov_blend):
    c = corridor
    kw = dict(WIDE, trans_thresh=0.3, rot_thresh=0.2, cov_blend=cov_blend)
    starts = [10, 100, 250, 400]
    beams = [360, 1080, 180, 720]
    fleets = [_fleet(gpu_api, c, 4, **kw) for _ in range(3)]
    for f in fleets:
        for r, t in enumerate(starts):
            f.setPose(r, *c["data"][beams[r]]["truth"][t])
    for i in range(12):
        for f, rs in zip(fleets, ([2], [0, 1, 2, 3], [3, 2, 1, 0])):
            b = [beams[r] for r in rs]
            f.update(rs, [c["data"][bb]["scans"][starts[r] + i] for r, bb in zip(rs, b)], [c["data"][bb]["odom"][starts[r] + i] for r, bb in zip(rs, b)],
                     force=[i == 0] * len(rs))
        got = [f._get() for f in fleets]
        for a, b in zip(got[0], got[1]):
            assert (a[2] == b[2]).all(), i                  # robot 2 alone == robot 2 in the full batch
        for a, b in zip(got[1], got[2]):
            assert (a == b).all(), i                        # the order of a batch does not show


def test_global_localization_in_one_launch(gpu_api, po, corridor):
    c = corridor
    kw = dict(KW, gloc_particles=3000)
    dev = dict(dir_dim=16, max_beams=512, timing=1)
    R = 4
    f = _fleet(gpu_api, c, R, follow=True, **dev, **kw)
    hs = [_single(gpu_api, c, follow=True, **dev, **kw) for _ in range(R)]
    ols = [_oracle(po, c, **kw) for _ in range(R)]
    free = _free(84.0)
    f.occupancySet(free, -1)
    f.occupancySet(c["cells"], 1)
    for r in range(R):
        hs[r].occupancySet(free, -1)
        hs[r].occupancySet(c["cells"], 1)
        ols[r].occ_set(free, -1)
        ols[r].occ_set(c["cells"], 1)
    starts = [100, 160, 220, 30]
    truth = c["data"][360]["truth"]
    for r, t in enumerate(starts):
        x, y, a = truth[t]
        p = (x - 30.0, y, a + 1.0) if r < 3 else (x, y, a)   # robots 0-2 start lost, robot 3 tracks
        f.setPose(r, *p)
        hs[r].setPose(*p)
        ols[r].set_pose(*p)
        hs[r].first = True
    for r in range(3):
        for h in (f,):
            h.setSeed(r, 91 + r)
            h.triggerGlobalLocalization(r)
        hs[r].setSeed(91 + r)
        hs[r].triggerGlobalLocalization()
        ols[r].set_seed(91 + r)
        ols[r].trigger_global_localization()
    assert f.distance_map.window()["parked"] > 0
    gloc_rounds = 0
    for i in range(40):
        before = f.distance_map.kernelTimes()[1]["match"]
        active = any(f.globalLocalizationActive(r) for r in range(3))
        _run(f, hs, ols, c, [[(r, starts[r] + i) for r in range(R)]])
        for h in hs:
            h.first = False
        launches = f.distance_map.kernelTimes()[1]["match"] - before
        assert launches <= 2, (i, launches)           # the candidates of every robot in one launch, then one tracking launch
        if launches == 2:
            assert active, i
            gloc_rounds += 1
        if not any(f.globalLocalizationActive(r) for r in range(3)):
            break
    assert gloc_rounds >= 1
    assert not any(f.globalLocalizationActive(r) for r in range(3))


def test_large_map_extent_path(gpu_api, po, corridor):
    c = corridor
    R = 8
    starts = [0, 60, 120, 180, 260, 340, 420, 500]   # spread over the whole corridor, out and back
    f16 = _fleet(gpu_api, c, R, follow=True, dir_dim=16, max_beams=512, **KW)
    f128 = _fleet(gpu_api, c, R, dir_dim=128, max_beams=512, **KW)
    hs = [_single(gpu_api, c, dir_dim=128, max_beams=512, **KW) for _ in range(R)]   # a fixed window that holds the whole corridor
    _place(f16, hs, None, starts, c)
    for r, t in enumerate(starts):
        f128.setPose(r, *c["data"][360]["truth"][t])
    assert f16.distance_map.window()["parked"] > 0
    shifts = f16.distance_map.window()["shifts"]
    plan = [[(r, starts[r] + i) for r in range(R)] for i in range(16)]
    data = c["data"][360]

    def also_128(i):
        rs = list(range(R))
        f128.update(rs, [data["scans"][starts[r] + i] for r in rs], [data["odom"][starts[r] + i] for r in rs], force=[r == 0 and i == 0 for r in rs])

    _run(f16, hs, None, c, plan, before_round=also_128)
    for a, b in zip(f16._get(), f128._get()):
        assert (a == b).all()
    assert f16.distance_map.window()["shifts"] == shifts   # the fleet never moves the window
    assert f16.distance_map.window()["parked"] > 0


def test_map_edits_between_rounds(gpu_api, po, corridor):
    c = corridor
    R = 4
    starts = [20, 60, 140, 200]
    f = _fleet(gpu_api, c, R, **WIDE, **KW)
    hs = [_single(gpu_api, c, **WIDE, **KW) for _ in range(R)]
    _place(f, hs, None, starts, c)
    O = 1321122 * 32
    rng = np.random.default_rng(8)
    edits = {}
    for i in (3, 6, 9):
        x0 = int((5.0 + 3 * i) * 20) + O
        k = np.sort(rng.choice(60 * 31, 150, replace=False))
        edits[i] = np.stack([x0 + k // 31, O - 15 + k % 31], 1).astype(np.uint32)

    def edit(i):
        if i in edits:
            for m in [f.distance_map] + [h.distance_map for h in hs]:
                m.addObstacle(edits[i])
                if i == 9:
                    m.removeObstacle(edits[3][::2])
                m.update()

    _run(f, hs, None, c, [[(r, starts[r] + i) for r in range(R)] for i in range(14)], before_round=edit)


def test_bad_arguments_change_nothing(gpu_api, po, corridor):
    c = corridor
    f = _fleet(gpu_api, c, 3, **WIDE, max_beams=512, **KW)
    d = c["data"][360]
    for r in range(3):
        f.setPose(r, *d["truth"][10 * r])
    f.update([0, 1, 2], [d["scans"][10 * r] for r in range(3)], [d["odom"][10 * r] for r in range(3)], force=[1, 1, 1])
    ref = f._get()
    s, o = d["scans"][40], d["odom"][40]
    bad = [([0, 3], [s, s], [o, o]),                       # out of range
           ([-1], [s], [o]),
           ([1, 1], [s, s], [o, o]),                       # repeated
           ([0, 2], [s, np.zeros((513, 3))], [o, o]),      # over max_beams
           ([0, 2], [s, np.zeros((0, 3))], [o, o])]        # empty
    for rs, sc, od in bad:
        with pytest.raises(gpu_api.LamaError) as e:
            f.update(rs, sc, od, force=[1] * len(rs))
        assert e.value.code == -1, rs
        for a, b in zip(ref, f._get()):
            assert (a == b).all(), rs
