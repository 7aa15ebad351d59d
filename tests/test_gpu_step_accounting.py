"""Step accounting of the 2-D front ends, pinned scan by scan: kernel launch counts (kernelTimes), host <-> device bytes (traffic) and
the last scan's work counters, for every way a scan reaches the device's match and map update:

- Slam2D: match + update_maps;
- PFSlam2D in timing mode: match + update_maps_async on one stream;
- PFSlam2D at 256 particles with one group: the pipelined single-stream step;
- PFSlam2D at 256 particles with four groups: the grouped step;
- two logical sharded ranks on one device in timing mode: shard_begin, shard_map_update and update_maps_async.

The expected values are in tests/golden/step_accounting.json.  `detached` is left out where several particles share patches: two
particles that write a patch they share in the same update copy it once or twice as their CTAs happen to finish
(tests/test_gpu_pf_groups.py).  The three 256-particle filters must also agree bit for bit on states, weights and resampling history."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_accounting.json")
PF_KW = dict(trans_thresh=0.05, rot_thresh=0.05, seed=42, meas_sigma_gain=0.0008)
SCANS = 36


def _record(h, traffic=True, detached=True):
    """what one scan left: counters() and traffic() first (both settle), then the launch counts"""
    last, _ = h.counters()
    if not detached:
        last = {k: v for k, v in last.items() if k != "detached"}
    r = dict(counters=last)
    if traffic:
        r["traffic"] = list(h.traffic())
    ms, launches = h.kernelTimes()
    r["launches"] = launches
    return r, ms


def _timed(ms):
    return ms["match_ms"] > 0 and ms["raycast_ms"] > 0 and ms["brushfire_ms"] > 0


def run_slam(api, synth):
    ds = synth.make_dataset("room", SCANS, n_beams=1080)
    h = api.Slam2D(api.Slam2D.Options(timing=1))
    h.setPose(*ds.truth[0])
    recs = []
    for t in range(SCANS):
        h.update(ds.scans[t], ds.odom[t])
        r, ms = _record(h, traffic=False)
        recs.append(r)
    return recs, ms


def run_pf(api, synth, groups=None, timing=0):
    """256 particles on the loop; LAMA_PF_GROUPS is read when the engine is created by the first update"""
    ds = synth.make_dataset("loop", SCANS, n_beams=1080)
    h = api.PFSlam2D(api.PFSlam2D.Options(256, timing=timing, **PF_KW))
    h.setPrior(*ds.truth[0])
    old = os.environ.pop("LAMA_PF_GROUPS", None)
    if groups is not None:
        os.environ["LAMA_PF_GROUPS"] = str(groups)
    try:
        h.update(ds.scans[0], ds.odom[0])
    finally:
        os.environ.pop("LAMA_PF_GROUPS", None)
        if old is not None:
            os.environ["LAMA_PF_GROUPS"] = old
    recs, states = [], []
    for t in range(SCANS):
        if t:
            h.update(ds.scans[t], ds.odom[t])
        s, w = h.getParticles()
        states.append((s, w, h.resampleDigest()))
        r, ms = _record(h, detached=False)
        recs.append(r)
    return recs, ms, states


def run_shards(api, synth):
    from iris_lama_b200.distributed import LocalShards
    P, G = 32, 2
    ds = synth.make_dataset("room", SCANS, n_beams=360)
    opts = dict(trans_thresh=0.05, rot_thresh=0.05, seed=7, meas_sigma_gain=0.002, timing=1)
    hs = [api.PFSlam2D(api.PFSlam2D.Options(P, shard_rank=r, shard_count=G, **opts)) for r in range(G)]
    for h in hs:
        h.setPrior(*ds.truth[0])
    sh = LocalShards(hs, P)
    recs, ms = [], []
    for t in range(SCANS):
        sh.update(ds.scans[t], ds.odom[t])
        rr = [_record(h, detached=False) for h in hs]
        recs.append([r for r, _ in rr])
        ms = [m for _, m in rr]
    return recs, ms


def run_all(api, synth):
    """every case's per-scan records (the contents of the golden file) and what the test checks beside them"""
    slam, slam_ms = run_slam(api, synth)
    pf_t, pf_t_ms, st_t = run_pf(api, synth, timing=1)
    pf_1, _, st_1 = run_pf(api, synth, groups=1)
    pf_4, _, st_4 = run_pf(api, synth, groups=4)
    shards, shard_ms = run_shards(api, synth)
    records = dict(slam2d=slam, pf_timing=pf_t, pf_one_group=pf_1, pf_four_groups=pf_4, shards=shards)
    return records, dict(timed=[slam_ms, pf_t_ms] + shard_ms, states=(st_t, st_1, st_4))


@pytest.fixture(scope="module")
def runs(gpu_api, synth):
    return run_all(gpu_api, synth)


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", ["slam2d", "pf_timing", "pf_one_group", "pf_four_groups", "shards"])
def test_step_accounting(runs, golden, case):
    got, want = runs[0][case], golden[case]
    assert len(got) == len(want)
    for t, (g, w) in enumerate(zip(got, want)):
        assert g == w, (case, t)


def test_timing_mode_times_every_kernel(runs):
    for ms in runs[1]["timed"]:
        assert _timed(ms), ms


def test_one_stream_and_groups_agree(runs):
    st_t, st_1, st_4 = runs[1]["states"]
    for t, (a, b, c) in enumerate(zip(st_t, st_1, st_4)):
        for o in (b, c):
            assert (o[0] == a[0]).all() and (o[1] == a[1]).all(), t
            assert o[2] == a[2], t
    assert st_t[-1][2][0] >= 2   # the filter resampled
