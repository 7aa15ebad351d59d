"""Checkpoints of GraphSlam2D sessions (lama_graph_save_state / lama_graph_load_state, file kind 4, DESIGN.md §13).

A GraphSlam2D saved at any point of a run, loaded and continued, must report exactly what the uninterrupted run reports: key poses
and clouds, links, loop candidates, statistics, the inner Slam2D and the global maps generated later.  The CPU tests write the documented
kind-4 layout with an independent Python writer and check the reader: valid files load (LAMA_ERR_NO_DEVICE without a GPU), every
corruption gives LAMA_ERR_ARG and no handle."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

from test_checkpoint import _slam_state, frame, slam_payload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, ERR_ARG, ERR_NO_DEVICE = 0, -1, -3
KIND = 4
SE2_ID = struct.pack("<4d", 1.0, 0.0, 0.0, 0.0)
HOT, OWN = 1 << 28, 1 << 29


# ---- an independent writer of the kind-4 layout ----------------------------------------------------------------------------------
def se2(x, y, r):
    return struct.pack("<4d", math.cos(r), math.sin(r), x, y)


def graph_options(head_delay=5, max_candidates=5, ignore_n=20, key_distance=1.0, key_angle=0.5 * math.pi):
    return (struct.pack("<ddi", key_distance, key_angle, head_delay) + struct.pack("<ddi", 10.0, 2.0, max_candidates)
            + struct.pack("<dii", 0.05, 10, ignore_n))


def inner_slam(has_first, transient=1, truncated_ray=1.0, occupancy=0, lidar=0, dir_dim=8):
    """the options and state bytes of a kind-2 file, with the options GraphSlam2D forces"""
    b = struct.pack("<6d", 0.5, 0.5, 0.5, truncated_ray, 0.0, 0.05) + struct.pack("<IIii", 32, 100, 0, occupancy)
    b += bytes([transient, lidar]) + struct.pack("<iii", dir_dim, 0, 2048)
    b += SE2_ID * 3 + bytes([has_first, has_first]) + struct.pack("<IQQ", 7, 0, 3) + struct.pack("<6Q", *range(6)) * 2
    return b


def graph_state(correction=SE2_ID, mapping_keyid=0, candidates=(), center=(0.0, 0.0), stats=(0, 0, 0), report=(-1, 0, 0, 0, 0.0, 0.0, 0.0)):
    b = correction + se2(1e10, 1e10, 0.0) + struct.pack("<2d", 0.0, 0.0) + struct.pack("<Q", mapping_keyid)
    b += struct.pack("<3Q", *stats) + struct.pack("<iIIQ3d", *report)
    b += struct.pack("<I", len(candidates)) + struct.pack(f"<{len(candidates)}i", *candidates) + struct.pack("<2d", *center)
    return b


def key_pose(i, n_pts=4, pose=None, quat=(0.0, 0.0, 0.0, 1.0), key_id=None, m_field=None):
    p = se2(0.5 * i, 0.1 * i, 0.05 * i) if pose is None else pose
    b = struct.pack("<i", i if key_id is None else key_id) + p + p + struct.pack("<3d", 0.1, 0.0, 0.2) + struct.pack("<4d", *quat)
    b += struct.pack("<d", float(i)) + struct.pack("<I", n_pts if m_field is None else m_field)
    return b + (np.arange(3 * n_pts, dtype=np.float64) * 0.25 + i).tobytes()


def loss(sigma, k):
    return struct.pack("<4d", *sigma, k)


def factors(items):
    return struct.pack("<I", len(items)) + b"".join(struct.pack("<ii", a, b) + se2(0.5, 0.1, 0.05) + loss(s, k) for a, b, s, k in items)


def engine(dir_dim=8, pool=16, known_plane=False, kind=0, particles=1, refcount=(1, 1), res=0.05, l2=0.5):
    """an engine section followed by its slot payloads: slot 0 the occupancy patch at entry 10, slot 1 the distance patch"""
    K = len(refcount)
    b = b"\x01" + struct.pack("<5i", particles, dir_dim, pool, 2048, kind) + bytes([1 if known_plane else 0])
    b += struct.pack("<2d", res, l2) + struct.pack("<2i", 1321122 - dir_dim // 2, 1321122 - dir_dim // 2)
    b += struct.pack("<3QI", K, 0, 0, K) + struct.pack(f"<{K}i", *refcount)
    dirs = np.full((particles, 3 if kind == 1 else 2, dir_dim * dir_dim), -1, np.int32)
    dirs[0, 0, 10] = 0 | HOT
    if K > 1:
        dirs[0, 1, 10] = 1 | OWN
    b += dirs.tobytes()
    stride = 4096 + 128 + (128 if known_plane or kind == 1 else 0)
    return b + np.random.default_rng(K + dir_dim).integers(0, 256, size=K * stride, dtype=np.uint8).tobytes()


def fresh_payload():
    """a GraphSlam2D saved before its first update: no keys, no engines"""
    return (graph_options() + inner_slam(0) + graph_state() + struct.pack("<I", 0) + struct.pack("<I", 0)
            + struct.pack("<I", 0) + factors([]) + factors([]) + b"\x00" + b"\x00")


def graph_payload(opts=None, slam=None, keys=None, links=((0, 2),), priors=None, chain=None, queue=None, candidates=(0,), mapping_keyid=3,
                  inner=None, glob=None, trailing=b""):
    """three keys, a link, the prior, two chain factors, one queued loop factor, an inner engine and the known-plane global map"""
    b = graph_options() if opts is None else opts
    b += inner_slam(1) if slam is None else slam
    b += graph_state(correction=se2(0.02, -0.01, 0.003), mapping_keyid=mapping_keyid, candidates=candidates, center=(3.0, -2.0),
                     stats=(1, 1, 1), report=(0, 4, 5, 37, 2.5, 0.01, 0.7))
    ks = [key_pose(i) for i in range(3)] if keys is None else keys
    b += struct.pack("<I", len(ks)) + b"".join(ks)
    b += struct.pack("<I", len(links)) + b"".join(struct.pack("<ii", a, c) for a, c in links)
    pr = [(0, (0.01, 0.01, 0.01), 0.0)] if priors is None else priors
    b += struct.pack("<I", len(pr)) + b"".join(struct.pack("<i", n) + se2(0, 0, 0) + loss(s, k) for n, s, k in pr)
    b += factors([(0, 1, (0.25, 0.25, 0.15), 0.0), (1, 2, (0.25, 0.25, 0.15), 0.0)] if chain is None else chain)
    b += factors([(0, 2, (1.0, 1.0, 1.0), 0.1)] if queue is None else queue)
    b += engine() if inner is None else inner
    b += (engine(pool=64, known_plane=True, refcount=(1,), l2=0.05) if mapping_keyid else b"\x00") if glob is None else glob
    return b + trailing


def _load(api, path, fn="graph", dev=None):
    L = api.lib()
    f = {"graph": L.lama_graph_load_state, "slam": L.lama_slam_load_state, "pf": L.lama_pf_load_state}[fn]
    h = C.c_void_p()
    rc = f(str(path).encode(), C.byref(dev) if dev is not None else None, C.byref(h))
    return rc, h


def _destroy(api, fn, h):
    L = api.lib()
    {"graph": L.lama_graph_destroy, "slam": L.lama_slam_destroy, "pf": L.lama_pf_destroy}[fn](h)


def _expect_valid(api, path):
    rc, h = _load(api, path)
    if api.device_count() < 1:
        assert rc == ERR_NO_DEVICE, (rc, api.lib().lama_last_error())
        assert not h.value
    else:
        assert rc == OK, api.lib().lama_last_error()
        _destroy(api, "graph", h)


def _expect_bad(api, path, fn="graph", dev=None, msg=None):
    L = api.lib()
    rc, h = _load(api, path, fn, dev)
    assert rc == ERR_ARG, (rc, L.lama_last_error())
    assert not h.value
    if msg:
        assert msg in L.lama_last_error().decode(), L.lama_last_error()


def test_python_written_files_are_read(api, tmp_path):
    for name, data in [("fresh", frame(fresh_payload(), kind=KIND)), ("full", frame(graph_payload(), kind=KIND)),
                       ("no_global", frame(graph_payload(mapping_keyid=0), kind=KIND)),
                       ("no_points", frame(graph_payload(keys=[key_pose(i, n_pts=0) for i in range(3)]), kind=KIND)),
                       ("no_angular_key_test", frame(graph_payload(opts=graph_options(key_angle=math.inf)), kind=KIND))]:
        p = tmp_path / f"{name}.ckpt"
        p.write_bytes(data)
        _expect_valid(api, p)


def test_loaded_options_are_the_saved_ones(api, tmp_path):
    """GraphSlam2D.loadState describes the session with the options the file holds, and the device of the call"""
    p = tmp_path / "o.ckpt"
    p.write_bytes(frame(graph_payload(opts=graph_options(head_delay=3, key_angle=math.inf)), kind=KIND))
    o = api._graph_options_of_checkpoint(p, 1, 7, True)
    assert (o.key_pose_distance, o.key_pose_angular_distance, o.key_pose_head_delay, o.loop_search_max_distance) == (1.0, math.inf, 3, 10.0)
    assert (o.loop_closure_scan_rmse, o.loop_closure_max_candidates, o.ignore_n_chain_poses) == (0.05, 10, 20)
    s = o.slam
    assert (s.truncated_ray, s.resolution, s.patch_size, s.occupancy, s.transient_map, s.lidar_odometry) == (1.0, 0.05, 32, 0, 1, 0)
    assert (s.dev.dir_dim, s.dev.pool_slots, s.dev.max_beams, s.dev.device, s.dev.stream, s.dev.timing) == (8, 0, 2048, 1, 7, 1)


@pytest.mark.parametrize("cut", [0, 7, 31, 33, 120, 0.5, -9000, -4300, -1])
def test_truncated_files_are_refused(api, tmp_path, cut):
    data = frame(graph_payload(), kind=KIND)
    cut = int(len(data) * cut) if isinstance(cut, float) else cut
    p = tmp_path / "t.ckpt"
    p.write_bytes(data[:cut] if cut >= 0 else data[:len(data) + cut])
    _expect_bad(api, p)


def test_flipped_byte_and_bad_version_are_refused(api, tmp_path):
    data = bytearray(frame(graph_payload(), kind=KIND))
    p = tmp_path / "h.ckpt"
    for off in (40, len(data) // 3, len(data) - 10):
        flipped = bytearray(data)
        flipped[off] ^= 0x10
        p.write_bytes(bytes(flipped))
        _expect_bad(api, p, msg="checksum")
    p.write_bytes(frame(graph_payload(), kind=KIND, version=2))
    _expect_bad(api, p, msg="version")


NAN = float("nan")
CORRUPTIONS = {   # case: (writer arguments, a part of the refusal message)
    "key_id": (dict(keys=[key_pose(0), key_pose(1, key_id=5), key_pose(2)]), "id differs"),
    "nonfinite_pose": (dict(keys=[key_pose(0), key_pose(1, pose=se2(NAN, 0, 0)), key_pose(2)]), "non-finite"),
    "nonfinite_quat": (dict(keys=[key_pose(0), key_pose(1, quat=(0, 0, NAN, 1)), key_pose(2)]), "non-finite"),
    "point_count": (dict(keys=[key_pose(0), key_pose(1, m_field=1 << 28), key_pose(2)]), "key points"),
    "prior_node": (dict(priors=[(3, (0.01, 0.01, 0.01), 0.0)]), "prior names no key"),
    "factor_node": (dict(chain=[(0, 1, (0.25, 0.25, 0.15), 0.0), (1, 3, (0.25, 0.25, 0.15), 0.0)]), "names no key"),
    "queue_node": (dict(queue=[(-1, 2, (1.0, 1.0, 1.0), 0.1)]), "names no key"),
    "link_node": (dict(links=((0, 9),)), "link names no key"),
    "candidate": (dict(candidates=(0, 3)), "candidate names no key"),
    "zero_sigma": (dict(chain=[(0, 1, (0.25, 0.0, 0.15), 0.0), (1, 2, (0.25, 0.25, 0.15), 0.0)]), "bad loss"),
    "negative_sigma": (dict(priors=[(0, (0.01, -0.01, 0.01), 0.0)]), "bad loss"),
    "negative_huber": (dict(queue=[(0, 2, (1.0, 1.0, 1.0), -0.1)]), "bad loss"),
    "mapping_keyid_past_keys": (dict(mapping_keyid=4), "mapping key id"),
    "global_without_mapping_keyid": (dict(mapping_keyid=0, glob=engine(pool=64, known_plane=True, refcount=(1,), l2=0.05)), "present exactly"),
    "mapping_keyid_without_global": (dict(mapping_keyid=3, glob=b"\x00"), "present exactly"),
    "global_two_particles": (dict(glob=engine(pool=64, known_plane=True, particles=2, refcount=(1,), l2=0.05)), "particle count"),
    "global_logodds": (dict(glob=engine(pool=64, kind=1, refcount=(1,), l2=0.05)), "occupancy kind"),
    "global_without_known_plane": (dict(glob=engine(pool=64, known_plane=False, refcount=(1,), l2=0.05)), "known plane"),
    "inner_not_transient": (dict(slam=inner_slam(1, transient=0)), "forces"),
    "inner_truncated_ray": (dict(slam=inner_slam(1, truncated_ray=0.0)), "forces"),
    "inner_logodds": (dict(slam=inner_slam(1, occupancy=1)), "forces"),
    "inner_lidar_odometry": (dict(slam=inner_slam(1, lidar=1)), "bad options"),
    "keys_without_inner_engine": (dict(inner=b"\x00"), "without device state"),
    "negative_ignore_n": (dict(opts=graph_options(ignore_n=-1)), "bad graph options"),
    "nan_graph_option": (dict(opts=graph_options(key_distance=NAN)), "bad graph options"),
    "infinite_sigma": (dict(chain=[(0, 1, (0.25, math.inf, 0.15), 0.0), (1, 2, (0.25, 0.25, 0.15), 0.0)]), "bad loss"),
    "trailing": (dict(trailing=b"\x00"), "bytes after"),
}


def test_nonfinite_correction_is_refused(api, tmp_path):
    b = bytearray(graph_payload())
    off = len(graph_options()) + len(inner_slam(1))          # the correction opens the graph state
    b[off + 16:off + 24] = struct.pack("<d", math.inf)       # its x
    p = tmp_path / "c.ckpt"
    p.write_bytes(frame(bytes(b), kind=KIND))
    _expect_bad(api, p, msg="non-finite")


@pytest.mark.parametrize("case", sorted(CORRUPTIONS))
def test_semantic_corruptions_with_a_valid_checksum_are_refused(api, tmp_path, case):
    p = tmp_path / "c.ckpt"
    kw, msg = CORRUPTIONS[case]
    p.write_bytes(frame(graph_payload(**kw), kind=KIND))
    _expect_bad(api, p, msg=msg)


def test_wrong_kinds_are_refused(api, tmp_path):
    g = tmp_path / "graph.ckpt"
    g.write_bytes(frame(graph_payload(), kind=KIND))
    _expect_bad(api, g, fn="slam", msg="GraphSlam2D")
    _expect_bad(api, g, fn="pf", msg="GraphSlam2D")
    for kind, lidar in ((1, False), (2, False), (3, True)):   # the graph loader refuses by kind, before it parses the body
        p = tmp_path / f"k{kind}.ckpt"
        p.write_bytes(frame(slam_payload(lidar=lidar), kind=kind))
        _expect_bad(api, p, msg="not a GraphSlam2D")


def test_geometry_is_checked(api, tmp_path):
    p = tmp_path / "g.ckpt"
    p.write_bytes(frame(graph_payload(), kind=KIND))
    for field, v in [("dir_dim", 16), ("pool_slots", 17), ("max_beams", 1080)]:
        dev = api.DeviceOptions(device=0, dir_dim=0, pool_slots=0, max_beams=0, timing=0, stream=0)
        setattr(dev, field, v)
        _expect_bad(api, p, dev=dev, msg="geometry")
    dev = api.DeviceOptions(device=0, dir_dim=8, pool_slots=16, max_beams=2048, timing=0, stream=0)   # the saved values are accepted
    rc, h = _load(api, p, dev=dev)
    assert rc == (OK if api.device_count() else ERR_NO_DEVICE), api.lib().lama_last_error()
    _destroy(api, "graph", h)


def test_new_entry_points_refuse_null_arguments(api, tmp_path):
    L = api.lib()
    null = C.c_void_p(None)
    h = C.c_void_p()
    path = str(tmp_path / "x.ckpt").encode()
    for fn, args in [(L.lama_graph_save_state, (null, path)), (L.lama_graph_save_state, (null, null)),
                     (L.lama_graph_load_state, (null, null, C.byref(h))), (L.lama_graph_load_state, (path, null, null))]:
        assert fn(*args) == ERR_ARG, fn.__name__
        assert b"null" in L.lama_last_error()
    assert not h.value


def test_header_compiles_as_c99_with_the_new_entry_points(tmp_path):
    src = tmp_path / "c99.c"
    src.write_text('#include "lama_b200.h"\n'
                   'int f(lama_graph* g, lama_graph** out) { return lama_graph_save_state(g, "a") + lama_graph_load_state("a", 0, out); }\n')
    subprocess.check_call(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])


# ---- GPU: continuation == uninterrupted run ---------------------------------------------------------------------------------------
N_SCANS = 1600
QUIET = 30   # the global-map cases: scans after the save with new keys and no optimisation, so the next generateOccupancyMap is incremental


@pytest.fixture(scope="module")
def loop_run(synth):
    """two laps of the 30 m room, and the save points chosen by inspecting an uninterrupted run: after scan t (0-based), the key count,
    the loop factors, the optimisations and whether a loop factor is queued"""
    from iris_lama_b200 import api
    ds = synth.make_dataset("loop", N_SCANS, n_beams=1080)
    g = api.GraphSlam2D()
    g.Init(*ds.truth[0])
    rows, flushed = [], 0
    for t in range(N_SCANS):
        g.update(ds.scans[t], ds.odom[t], float(t))
        st = g.stats()
        if st["optimizations"] > (rows[-1]["optimizations"] if rows else 0):
            flushed = st["loop_factors"]
        rows.append(dict(st, queued=st["loop_factors"] - flushed))
    ignore_n = g.options.ignore_n_chain_poses
    opt_at = [t for t in range(1, N_SCANS) if rows[t]["optimizations"] > rows[t - 1]["optimizations"]]
    ok_at = [t for t in opt_at if rows[t]["optimizations_ok"] > rows[t - 1]["optimizations_ok"]]
    assert len(ok_at) >= 2 and rows[-1]["loop_factors"] >= 5, (opt_at, rows[-1])

    def quiet(k, n):   # no optimisation in scans k .. k + n - 1, and new keys meanwhile
        return all(rows[t]["optimizations"] == rows[k - 1]["optimizations"] for t in range(k, k + n)) and rows[k + n - 1]["key_poses"] > rows[k - 1]["key_poses"]

    points = {"fresh": 0}
    points["early"] = next(t + 1 for t in range(N_SCANS) if 0 < rows[t]["key_poses"] < ignore_n and rows[t]["key_poses"] >= ignore_n // 2)
    # a loop factor queued, and optimised later in the continuation
    points["queued"] = next(t + 1 for t in range(N_SCANS - 1) if rows[t]["queued"] > 0 and t + 1 not in opt_at and t not in opt_at)
    points["optimised"] = ok_at[0] + 1
    points["global_full"] = next(k for k in range(ok_at[0] + 2, N_SCANS - QUIET) if quiet(k, QUIET))
    points["global_coarse"] = next(k for k in range(ok_at[1] + 2, N_SCANS - QUIET) if quiet(k, QUIET))
    return ds, rows, points, opt_at


def _graph_state(g):
    cor, org, stamps = g.keyPoses()
    n = len(stamps)
    st = g.stats()
    rep = dict(st["last_report"])
    device_ms = rep.pop("device_ms")
    st = dict(st, last_report=rep)
    d = dict(pose=g.getPose().tobytes(), keys=(cor.tobytes(), org.tobytes(), stamps.tobytes()), links=g.links().tobytes(),
             cands=g.lastCandidates().tobytes(), stats=st, slam=_slam_state(g.slam, False))
    d["clouds"] = [tuple(a.tobytes() for a in g.keyCloud(i)) for i in sorted({0, n // 2, n - 1}) if n]
    return d, device_ms


def _global_maps(g, full):
    m = g.generateOccupancyMap(full=full)
    n, mn, mx = m.bounds()
    d = dict(res=m.resolution, bounds=(n, mn.tolist(), mx.tolist()))
    if n:
        d["cells"] = {k: v.tobytes() for k, v in m.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1])).items()}
    dm = g.generateCoarseDistanceMap()
    n, mn, mx = dm.bounds()
    d["coarse"] = (dm.processed, n, mn.tolist(), mx.tolist())
    if n:
        d["coarse_cells"] = {k: v.tobytes() for k, v in dm.export(int(mn[0]), int(mn[1]), int(mx[0] - mn[0]), int(mx[1] - mn[1])).items()}
    return d


CASES = ["fresh", "early", "queued", "optimised", "global_full", "global_coarse", "far"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_graph_continuation_equals_uninterrupted_run(gpu_api, loop_run, tmp_path, case):
    """A uninterrupted, S saved before scan k and continued, B loaded from S's file (and, in one case, its twin B2): all equal after
    every scan from k on; the global and coarse maps generated at the same moments on all of them are equal"""
    api = gpu_api
    ds, rows, points, opt_at = loop_run
    k = points["queued" if case == "far" else case]
    start = (150.0, -80.0, ds.truth[0][2]) if case == "far" else ds.truth[0]   # "far": a wrong window centre after the load breaks the maps
    A, S = api.GraphSlam2D(), api.GraphSlam2D()
    for h in (A, S):
        h.Init(*start)
    for t in range(k):
        assert A.update(ds.scans[t], ds.odom[t], float(t)) == S.update(ds.scans[t], ds.odom[t], float(t)), t
    full = case != "global_coarse"
    if case.startswith("global"):
        assert _global_maps(A, full) == _global_maps(S, full)   # the next call is incremental: it draws on the saved global map
    f1, f2 = tmp_path / "s.ckpt", tmp_path / "b.ckpt"
    S.saveState(f1)
    stats = api.checkpoint_stats()
    assert stats["file_bytes"] == os.path.getsize(f1)
    B = api.GraphSlam2D.loadState(f1)
    assert B.options.key_pose_head_delay == S.options.key_pose_head_delay and B.options.slam.transient_map == 1
    B.saveState(f2)                                            # compared at the end, after the maps that depend on the restored centre
    handles = [S, B] + ([api.GraphSlam2D.loadState(f1)] if case == "optimised" else [])
    if case.startswith("global"):
        assert stats["used_slots"] > 0 and rows[k - 1]["optimizations"] >= 1
    if case == "optimised":
        assert rows[k - 1]["optimizations_ok"] >= 1 and S.stats()["optimizations_ok"] >= 1
        assert np.abs(S.keyPoses()[0] - S.keyPoses()[1]).max() > 1e-6   # the correction is not the identity
    opts_at_save = S.stats()["optimizations"]
    # global maps a few updates after the save, then every 250 scans, and at the end
    gen_at = {k + QUIET - 1, N_SCANS - 1} | set(range(k + 250, N_SCANS, 250))
    ms_s = S.stats()["last_report"]["device_ms"]
    assert B.stats() == S.stats()
    for t in range(k, N_SCANS):
        did = {h.update(ds.scans[t], ds.odom[t], float(t)) for h in [A] + handles}
        assert len(did) == 1, t
        pa = A.getPose().tobytes()
        assert all(h.getPose().tobytes() == pa for h in handles), t
        if did.pop() or t == k:
            sa, _ = _graph_state(A)
            for h in handles:
                sh, ms = _graph_state(h)
                assert sh == sa, t
                if h is not S and h.stats()["optimizations"] == opts_at_save:
                    assert ms == ms_s, t                   # the restored report, until a new optimisation replaces it
        if t in gen_at:
            ga = _global_maps(A, full)
            assert all(_global_maps(h, full) == ga for h in handles), t
    assert f1.read_bytes() == f2.read_bytes()                  # canonical: save -> load -> save gives the same bytes
    st = A.stats()
    if case in ("queued", "far"):
        assert st["optimizations"] > opts_at_save and st["loop_factors"] > 0
    assert st["optimizations_ok"] >= 1


@pytest.mark.gpu
def test_refusals_of_real_files(gpu_api, loop_run, tmp_path):
    api = gpu_api
    ds, _, points, _ = loop_run
    g = api.GraphSlam2D()
    g.Init(*ds.truth[0])
    for t in range(points["early"]):
        g.update(ds.scans[t], ds.odom[t], float(t))
    p = tmp_path / "g.ckpt"
    g.saveState(p)
    _expect_bad(api, p, dev=api.DeviceOptions(device=0, dir_dim=32, pool_slots=0, max_beams=0, timing=0, stream=0), msg="geometry")
    _expect_bad(api, p, fn="slam", msg="GraphSlam2D")
    data = p.read_bytes()
    bad = tmp_path / "bad.ckpt"
    for cut in (16, 1000, len(data) // 2, len(data) - 1):
        bad.write_bytes(data[:cut])
        _expect_bad(api, bad)
    for off in (200, len(data) // 2, len(data) - 5000):
        flipped = bytearray(data)
        flipped[off] ^= 1
        bad.write_bytes(bytes(flipped))
        _expect_bad(api, bad, msg="checksum")
    bad.write_bytes(data[:8] + struct.pack("<I", 9) + data[12:])
    _expect_bad(api, bad, msg="version")
    bad.write_bytes(data + b"\x00")
    _expect_bad(api, bad)


SHIM_SRC = r'''
// a C++ caller through the shim: a small GraphSlam2D session, saved, loaded, both continued and compared
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <memory>
#include <vector>
#include "lama_b200_shim.hpp"
struct Q { double x() const {return 0;} double y() const {return 0;} double z() const {return 0;} double w() const {return 1;} };
struct Cloud { std::vector<std::array<double,3>> points; std::array<double,3> sensor_origin_{}; Q sensor_orientation_; };
struct Pose { double x_, y_, r_; double x() const {return x_;} double y() const {return y_;} double rotation() const {return r_;} };
static std::shared_ptr<Cloud> scan(double x)   // a 6 m x 4 m box seen from (x, 0)
{
  auto c = std::make_shared<Cloud>();
  for (int i = 0; i < 360; ++i) {
    const double a = i * 3.14159265358979323846 / 180.0, dx = std::cos(a), dy = std::sin(a);
    double t = 1e9;
    if (dx > 1e-9) t = std::min(t, (3.0 - x) / dx);
    if (dx < -1e-9) t = std::min(t, (-3.0 - x) / dx);
    if (dy > 1e-9) t = std::min(t, 2.0 / dy);
    if (dy < -1e-9) t = std::min(t, -2.0 / dy);
    c->points.push_back({t * dx, t * dy, 0.0});
  }
  return c;
}
static int keys(const lama_b200_shim::GraphSlam2D& g)
{
  int n = 0;
  lama_b200_shim::check(lama_graph_get_key_poses(g.handle(), nullptr, nullptr, nullptr, 0, &n));
  return n;
}
int main(int argc, char** argv) {
  (void)argc;
  auto o = lama_b200_shim::GraphSlam2D::defaults();
  o.slam.trans_thresh = 0.05; o.slam.rot_thresh = 0.05; o.key_pose_distance = 0.2;
  lama_b200_shim::GraphSlam2D a(o);
  a.Init(Pose{-1.5, 0, 0});
  for (int t = 0; t < 10; ++t) a.update(scan(-1.5 + 0.1 * t), Pose{0.1 * t, 0, 0}, t);
  a.generateOccupancyMap(true);
  a.saveState(argv[1]);
  auto b = lama_b200_shim::GraphSlam2D::loadState(argv[1]);
  if (keys(a) < 2 || keys(a) != keys(*b)) return 2;
  for (int t = 10; t < 25; ++t) {
    if (a.update(scan(-1.5 + 0.1 * t), Pose{0.1 * t, 0, 0}, t) != b->update(scan(-1.5 + 0.1 * t), Pose{0.1 * t, 0, 0}, t)) return 3;
    double pa[3], pb[3];
    a.getPose(pa); b->getPose(pb);
    if (pa[0] != pb[0] || pa[1] != pb[1] || pa[2] != pb[2] || keys(a) != keys(*b)) return 4;
  }
  a.generateOccupancyMap(false);
  b->generateOccupancyMap(false);
  std::printf("shim graph checkpoints ok %d\n", keys(a));
  return 0;
}
'''


def _build_shim(tmp_path):
    src = tmp_path / "graph_ckpt.cpp"
    src.write_text(SHIM_SRC)
    exe = tmp_path / "graph_ckpt"
    lib_dir = os.path.join(ROOT, "iris_lama_b200")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", lib_dir,
                           "-llama_b200", f"-Wl,-rpath,{lib_dir}"])
    return exe


def test_shim_graph_checkpoint_caller_compiles(api, tmp_path):
    _build_shim(tmp_path)


@pytest.mark.gpu
def test_shim_caller_saves_and_loads_a_graph(gpu_api, tmp_path):
    exe = _build_shim(tmp_path)
    out = subprocess.run([str(exe), str(tmp_path / "graph.ckpt")], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "shim graph checkpoints ok" in out.stdout
