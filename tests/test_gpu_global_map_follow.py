"""A global map without an edge, on the device: a FrequencyOccupancyMap that follows its scans (Engine::render_scans in groups, each in
its own window, with a pool that grows) and GraphSlam2D's global map, which always follows.  Checked against the oracle render
(tests/global_map_oracle.py), whose map has no edge, and against the same render in a window that never moves."""
import math

import numpy as np
import pytest

import global_map_oracle as gmo
from test_global_map import _same_map, _state

pytestmark = pytest.mark.gpu

ERR_WINDOW, ERR_POOL = -4, -5


def _spread_scans(synth, n, seed, length, scale=(0.3, 0.6)):
    """n posed scans of the room dataset, shrunk, at random positions along `length` m of x and random headings"""
    rng = np.random.default_rng(seed)
    ds = synth.make_dataset("room", 2, n_beams=361)
    scans, states = [], []
    for k in range(n):
        scans.append(ds.scans[k % 2] * rng.uniform(*scale))
        states.append(_state(rng.uniform(0.0, length), rng.uniform(-4.0, 4.0), rng.uniform(-math.pi, math.pi)))
    return scans, np.array(states)


def _rounds(synth, length, res):
    out = []
    for rnd in range(4):
        scans, states = _spread_scans(synth, 16, seed=20 * rnd + int(res * 100), length=length)
        origins = np.tile([0.1, -0.05, 0.3], (len(scans), 1))
        quats = np.tile([0.0, 0.0, 0.0, 1.0], (len(scans), 1))
        if rnd == 2:   # tilted sensor: the 3-axis walk
            quats[::2] = [math.sin(0.05), 0.0, 0.0, math.cos(0.05)]
        out.append((scans, states, origins, quats, rnd != 1))
    return out


def _dump(m):
    n, mn, mx = m.bounds()
    e = m.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1]))
    return n, mn.tolist(), mx.tolist(), {k: v.tobytes() for k, v in e.items()}, m.exportImage().tobytes()


def test_following_map_over_300_m_equals_oracle(gpu_api, synth, tmp_path):
    """dir_dim 16, posed scans spread along 300 m in random order: every round's cell count, cells, bounds, patch set, query flags,
    and at the end the .sdm file and the image equal the oracle's; the window moved, parked and restored patches, the pool grew"""
    for res in (0.05, 0.1):
        g = gpu_api.FrequencyOccupancyMap(res, dir_dim=16, follow=True)
        o = gmo.OccupancyMap(res)
        assert g.pool()[0] == 256
        for rnd, (scans, states, origins, quats, full) in enumerate(_rounds(synth, 300.0, res)):
            assert g.insertScans(scans, states, full=full, origins=origins, quats=quats) == o.insert_scans(scans, states, full, origins=origins, quats=quats)
            _same_map(g, o, query=rnd == 0)
            g.prune(); o.prune()
            _same_map(g, o, tmp_path if rnd == 3 else None)
        w = g.window()
        slots, used = g.pool()
        assert w["shifts"] > 4 and w["parked"] > 0 and w["restored"] > 0, w
        assert slots > 256 and used > 256, (slots, used)


def test_following_changes_nothing_when_the_scans_fit_the_window(gpu_api, synth, tmp_path):
    """the same scans over 150 m in a dir_dim 128 window (205 m at 0.05 m): byte-identical exports, files and images with and without
    following, and no shift"""
    maps = [gpu_api.FrequencyOccupancyMap(0.05, dir_dim=128, max_beams=512, center=(75.0, 0.0), follow=f) for f in (False, True)]
    for scans, states, origins, quats, full in _rounds(synth, 150.0, 0.05):
        cells = {m.insertScans(scans, states, full=full, origins=origins, quats=quats) for m in maps}
        assert len(cells) == 1
        for m in maps:
            m.prune()
        assert _dump(maps[0]) == _dump(maps[1])
    a, b = tmp_path / "a.sdm", tmp_path / "b.sdm"
    maps[0].write(a)
    maps[1].write(b)
    assert a.read_bytes() == b.read_bytes()
    assert maps[1].window()["shifts"] == 0 and maps[1].pool() == maps[0].pool()


def test_a_scan_wider_than_the_window_is_refused_and_changes_nothing(gpu_api, synth):
    g = gpu_api.FrequencyOccupancyMap(0.05, dir_dim=8, follow=True)   # a 12.8 m window
    scans, states = _spread_scans(synth, 6, seed=4, length=40.0, scale=(0.2, 0.3))
    g.insertScans(scans, states, full=True)
    before, wb, pb = _dump(g), g.window(), g.pool()
    wide, _ = _spread_scans(synth, 1, seed=5, length=1.0, scale=(2.0, 2.0))
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertScans(scans[:3] + wide, np.concatenate([states[:3], states[:1]]), full=True)
    assert e.value.code == ERR_WINDOW and "scan 3" in str(e.value)
    assert _dump(g) == before and g.window() == wb and g.pool() == pb


def test_an_explicit_pool_is_a_hard_cap(gpu_api, synth):
    g = gpu_api.FrequencyOccupancyMap(0.05, dir_dim=16, pool_slots=64, follow=True)
    scans, states = _spread_scans(synth, 24, seed=6, length=300.0)
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertScans(scans, states, full=True)
    assert e.value.code == ERR_POOL
    assert g.pool() == (64, 64)


def _wide_out_and_back(synth, length, width, step=0.25, r_max=30.0, n_beams=360):
    """a corridor of `length` x `width` m driven to its far end and back, beams shorter than r_max (as test_gpu_window_follow's)"""
    segs = synth.make_corridor(length=length, width=width)
    xs = np.arange(0.0, length - 6.0, step)
    turn = np.linspace(0.0, np.pi, 10)[1:-1]
    path = [(x, 0.05 * np.sin(0.7 * x), 0.0) for x in xs] + [(xs[-1], 0.0, a) for a in turn]
    path += [(x, 0.05 * np.sin(0.7 * x), np.pi) for x in xs[::-1]]
    truth = np.array(path)
    angles = synth.beam_angles(n_beams, 360.0)
    rng_r, rng_o = np.random.default_rng(21), np.random.default_rng(22)
    scans, odom = [], np.zeros_like(truth)
    cur = tuple(truth[0])
    for t in range(len(truth)):
        r = synth.cast(segs, truth[t], angles, 40.0) + rng_r.normal(0.0, 0.01, n_beams)
        p = synth.scan_points(r, angles)
        scans.append(np.ascontiguousarray(p[np.hypot(p[:, 0], p[:, 1]) < r_max]))
        if t == 0:
            odom[0] = truth[0]
        else:
            d = synth._between(tuple(truth[t - 1]), tuple(truth[t]))
            cur = synth._compose(cur, (d[0] + rng_o.normal(0, 0.01), d[1] + rng_o.normal(0, 0.01), d[2] + rng_o.normal(0, 0.005)))
            odom[t] = cur
    return truth, odom, scans


def _graph_calls(g, ref, keyid, opts_seen, full):
    st = g.stats()
    if st["optimizations"] > opts_seen:   # mapping_keyid = 0 after every optimisation
        opts_seen, keyid = st["optimizations"], 0
    m = g.generateOccupancyMap(full=full)
    cor, _, _ = g.keyPoses()
    if keyid == 0:
        ref = gmo.OccupancyMap(0.05 if full else 0.1)
    new = range(keyid, len(cor))
    ref.insert_scans([g.keyCloud(i)[0] for i in new], [_state(*cor[i]) for i in new], full, thetas=cor[list(new), 2] if len(new) else None)
    ref.prune()
    return m, ref, len(cor), opts_seen


def test_graph_slam_global_map_follows_a_230_m_corridor(gpu_api, synth, tmp_path):
    """GraphSlam2D with default options (64 x 64 patches: 102.4 m at 0.05 m, 204.8 m at 0.1 m) out and back along a 230 m corridor 50 m
    wide: generateOccupancyMap every 150 scans with `full` alternating equals the oracle's render of the device's key poses and clouds
    after every call; a checkpoint taken while the global map has parked patches saves, loads and saves to the same bytes, and the
    resumed session's next global map equals the original's"""
    truth, odom, scans = _wide_out_and_back(synth, length=230.0, width=50.0)
    g = gpu_api.GraphSlam2D()
    g.Init(*truth[0])
    ref, keyid, opts_seen, calls, saved = None, 0, 0, 0, False
    most_patches, moved = 0, False
    for t in range(len(scans)):
        g.update(scans[t], odom[t], float(t))
        if t % 150 != 149 and t != len(scans) - 1:
            continue
        full = calls % 2 == 0
        calls += 1
        m, ref, keyid, opts_seen = _graph_calls(g, ref, keyid, opts_seen, full)
        _same_map(m, ref, tmp_path if calls == 6 else None, query=calls % 3 == 0)
        w = m.window()
        moved = moved or w["shifts"] > 0
        if full:
            most_patches = max(most_patches, m.bounds()[0])
        if not saved and w["parked"] > 0 and t > len(scans) // 2:
            saved = True
            a, b = tmp_path / "a.ckpt", tmp_path / "b.ckpt"
            g.saveState(a)
            r = gpu_api.GraphSlam2D.loadState(a)
            r.saveState(b)
            assert a.read_bytes() == b.read_bytes()
            assert r.generateOccupancyMap(full=full).window()["parked"] == w["parked"]
            for s in range(t + 1, min(t + 60, len(scans))):
                assert g.update(scans[s], odom[s], float(s)) == r.update(scans[s], odom[s], float(s)), s
            ma, mb = g.generateOccupancyMap(full=full), r.generateOccupancyMap(full=full)
            assert _dump(ma) == _dump(mb)
            del r
            break
    assert moved and saved and most_patches > 4096, (moved, saved, most_patches)
