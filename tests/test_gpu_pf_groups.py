"""PFSlam2D's step pipelined over particle groups (Engine::step_groups, DESIGN.md 7a) against the same filter on one stream: with G = 2,
3 and 4 groups (LAMA_PF_GROUPS, read when the engine is created; 4 is the default at 256 particles) every particle state, weight,
resampling decision and work counter, and every occupancy and distance cell of every particle must be equal bit for bit to G = 1.

`detached` is left out of the counter comparison: two particles that write a patch they share in the same update copy it once or
twice as their CTAs happen to finish, with or without groups (tests/test_gpu_window_follow.py)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KW = dict(trans_thresh=0.05, rot_thresh=0.05, seed=42)


def _handle(api, monkeypatch, groups, P, data, first, staged=None, **kw):
    """a filter whose engine is created with `groups` groups; the engine is made by the first update, so the variable is set around it"""
    monkeypatch.setenv("LAMA_PF_GROUPS", str(groups))
    o = dict(KW)
    o.update(kw)
    h = api.PFSlam2D(api.PFSlam2D.Options(P, **o))
    h.setPrior(*first)
    if staged is not None:
        h.stageScans(staged)
    h.update(data[0][0], data[0][1])
    monkeypatch.delenv("LAMA_PF_GROUPS")
    return h


def _step(h, t, scan, odom, staged):
    return h.updateStaged(t, odom) if staged else h.update(scan, odom)


def _no_detached(c):
    return {k: v for k, v in c.items() if k != "detached"}


def _assert_same_maps(a, b, P):
    for p in range(P):
        for kind in (0, 1):
            na, mna, mxa = a.mapBounds(p, kind)
            nb, mnb, mxb = b.mapBounds(p, kind)
            assert na == nb and (mna == mnb).all() and (mxa == mxb).all(), (p, kind)
        _, mn, mx = a.mapBounds(p, 0)
        w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
        oa, ob = a.exportOccupancy(p, int(mn[0]), int(mn[1]), w, h), b.exportOccupancy(p, int(mn[0]), int(mn[1]), w, h)
        for k in oa:
            assert (oa[k] == ob[k]).all(), (p, "occ", k)
        _, mn, mx = a.mapBounds(p, 1)
        w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
        da, db = a.exportDistance(p, int(mn[0]), int(mn[1]), w, h), b.exportDistance(p, int(mn[0]), int(mn[1]), w, h)
        for k in da:
            assert (da[k] == db[k]).all(), (p, "dm", k)


def _run(api, monkeypatch, P, scans, odom, first, groups=(2, 3, 4), staged_every=0, per_scan_counters=False, **kw):
    """G = 1 and each of `groups` over the same scans.  Host scans, or with staged_every = k every k-th scan from the staged copy (the
    others through host buffers, so both upload paths alternate).  States, weights and the resampling history are compared after every
    scan without a synchronising call in between, so the groups of consecutive scans overlap as they do in a run; with
    per_scan_counters the counters are read after every scan too (a barrier per scan)."""
    data = list(zip(scans, odom))
    staged = np.ascontiguousarray(np.stack(scans)) if staged_every else None
    hs = [_handle(api, monkeypatch, g, P, data, first, staged, **kw) for g in (1,) + tuple(groups)]
    resampled = 0
    for t in range(1, len(scans)):
        st = bool(staged_every) and t % staged_every == 0
        did = [_step(h, t, scans[t], odom[t], st) for h in hs]
        assert all(d == did[0] for d in did), t
        s0, w0 = hs[0].getParticles()
        d0 = hs[0].resampleDigest()
        for h in hs[1:]:
            s, w = h.getParticles()
            assert (s == s0).all() and (w == w0).all(), t
            assert h.resampleDigest() == d0, t
            assert (np.asarray(h.lastResample()) == np.asarray(hs[0].lastResample())).all(), t
        if per_scan_counters:
            c0 = hs[0].counters()[0]
            for h in hs[1:]:
                assert _no_detached(h.counters()[0]) == _no_detached(c0), t
        resampled = d0[0]
    t0 = hs[0].counters()[1]
    for h in hs[1:]:
        assert _no_detached(h.counters()[1]) == _no_detached(t0)
        assert h.getMemoryUsage()[1] == hs[0].getMemoryUsage()[1]
        _assert_same_maps(hs[0], h, P)
    return resampled


def test_groups_revisit_256x1080(gpu_api, monkeypatch, synth):
    """the benchmark's size: 256 particles x 1080 beams on the loop, the 300 scans that build the map and the first 60 of the revisit
    regime the benchmark times"""
    ds = synth.make_dataset("loop", 361, n_beams=1080)
    _run(gpu_api, monkeypatch, 256, ds.scans, ds.odom, ds.truth[0], staged_every=3, per_scan_counters=True)


def test_groups_forced_resampling(gpu_api, monkeypatch, synth):
    """meas_sigma_gain 0.0008: the filter resamples every few scans, so barriers, directory copies and k_merge_free run between grouped
    scans; 100 particles, which 3 groups split unevenly"""
    ds = synth.make_dataset("loop", 90, n_beams=1080)
    n = _run(gpu_api, monkeypatch, 100, ds.scans, ds.odom, ds.truth[0], staged_every=2, meas_sigma_gain=0.0008)
    assert n >= 3, n


def test_groups_window_shift(gpu_api, monkeypatch, synth):
    """a corridor driven further than a 16-patch window: window shifts, parked patches and their return between grouped scans"""
    segs = synth.make_corridor(length=84.0)
    xs = np.arange(0.0, 78.0, 0.3)
    truth = np.array([(x, 0.05 * np.sin(0.7 * x), 0.0) for x in xs] + [(x, 0.05 * np.sin(0.7 * x), np.pi) for x in xs[::-1]])
    angles = synth.beam_angles(360, 360.0)
    rng_r, rng_o = np.random.default_rng(11), np.random.default_rng(12)
    scans, odom = [], np.zeros_like(truth)
    cur = tuple(truth[0])
    for t in range(len(truth)):
        p = synth.scan_points(synth.cast(segs, truth[t], angles, 30.0) + rng_r.normal(0.0, 0.01, 360), angles)
        scans.append(np.ascontiguousarray(p[np.hypot(p[:, 0], p[:, 1]) < 8.0]))
        if t == 0:
            odom[0] = truth[0]
        else:
            d = synth._between(tuple(truth[t - 1]), tuple(truth[t]))
            cur = synth._compose(cur, (d[0] + rng_o.normal(0, 0.01), d[1] + rng_o.normal(0, 0.01), d[2] + rng_o.normal(0, 0.005)))
            odom[t] = cur
    data = list(zip(scans, odom))
    _run(gpu_api, monkeypatch, 16, scans, odom, truth[0], dir_dim=16, max_beams=512, seed=5, meas_sigma_gain=0.02)
    h = _handle(gpu_api, monkeypatch, 2, 16, data, truth[0], dir_dim=16, max_beams=512, seed=5, meas_sigma_gain=0.02)
    for t in range(1, len(scans)):
        h.update(scans[t], odom[t])
    w = h.window()
    assert w["shifts"] >= 3 and w["restored"] > 0 and w["parked"] > 0, w


@pytest.mark.parametrize("P,groups", [(2, (3,)), (5, (2, 4)), (37, (2, 3))])
def test_groups_uneven_and_fewer_particles(gpu_api, monkeypatch, synth, P, groups):
    """particle counts that G does not divide, and fewer particles than groups (the engine then uses one group per particle)"""
    ds = synth.make_dataset("room", 40, n_beams=1080)
    _run(gpu_api, monkeypatch, P, ds.scans, ds.odom, ds.truth[0], groups=groups, staged_every=2, meas_sigma_gain=0.05)
