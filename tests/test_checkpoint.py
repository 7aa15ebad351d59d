"""Checkpoints of PFSlam2D and Slam2D sessions (lama_*_save_state / lama_*_load_state, DESIGN.md §13).

A run that is saved after scan k, destroyed, loaded and continued must report exactly what the uninterrupted run reports, and saving must
not change the handle that is saved.  The CPU tests write the documented file layout with an independent Python writer and check the
reader: a valid file loads (LAMA_ERR_NO_DEVICE without a GPU), every corruption gives LAMA_ERR_ARG and no handle."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, ERR_ARG, ERR_NO_DEVICE, ERR_STATE = 0, -1, -3, -7
HDR = 32


# ---- an independent writer of the file layout ------------------------------------------------------------------------------------
def fnv1a64(b: bytes) -> int:
    h = 1469598103934665603
    for x in b:
        h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def frame(payload: bytes, kind=1, magic=b"LAMACKPT", version=1, total=None, checksum=None) -> bytes:
    total = HDR + len(payload) if total is None else total
    checksum = fnv1a64(payload) if checksum is None else checksum
    return magic + struct.pack("<IIQQ", version, kind, total, checksum) + payload


def mt19937_text(seed):
    mt = [seed & 0xFFFFFFFF]
    for i in range(1, 624):
        mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & 0xFFFFFFFF)
    return " ".join(str(v) for v in mt + [624]).encode()


SE2_ID = struct.pack("<4d", 1.0, 0.0, 0.0, 0.0)
HOT, OWN = 1 << 28, 1 << 29


def pf_payload(P=3, dir_dim=8, pool=16, refcount=(3, 1), entries=None, nodes=(-1,), node_of=None, rng=None, engine=True, trailing=b"",
               particles_field=None, engine_particles=None, K=None, flags_extra=0):
    """options, front-end state and the engine section of a PFSlam2D after its first scan: every particle shares slot 0 (occupancy,
    entry 10), particle 0 owns slot 1 (distance, entry 10)"""
    b = struct.pack("<I", P if particles_field is None else particles_field)
    b += struct.pack("<12d", 0.1, 0.2, 0.1, 0.2, 0.05, 3.0, 0.5, 0.5, 0.5, 0.0, 0.0, 0.05)
    b += struct.pack("<IIiiI", 32, 100, 0, -1, 42) + struct.pack("<iii", dir_dim, 0, 2048)
    b += SE2_ID + SE2_ID + (b"\x01" if engine else b"\x00") + struct.pack("<3d", 0.0, 0.0, float(P))
    b += SE2_ID * P + struct.pack(f"<{P}d", *([0.0] * P)) * 3
    b += struct.pack("<I", 0)                                    # no resampling in the last update
    b += struct.pack("<QQQ", 0, 1469598103934665603, 0)
    b += struct.pack("<I", 1) + struct.pack("<d", 0.0)           # getTimestamps
    b += struct.pack("<6Q", 1, 2, 3, 0, 0, 0) * 2 + struct.pack("<Q", 0) + struct.pack("<4d", 0.1, 0.2, 0.3, 0.4)
    b += struct.pack("<I", len(nodes)) + b"".join(SE2_ID + struct.pack("<i", p) for p in nodes)
    b += struct.pack(f"<{P}i", *(node_of if node_of is not None else [0] * P))
    r = mt19937_text(42) if rng is None else rng
    b += struct.pack("<I", len(r)) + r
    if not engine:
        return b + b"\x00" + trailing
    K = len(refcount) if K is None else K
    b += b"\x01" + struct.pack("<5i", P if engine_particles is None else engine_particles, dir_dim, pool, 2048, 0) + b"\x00"
    b += struct.pack("<2d", 0.05, 0.5) + struct.pack("<2i", 1321122 - dir_dim // 2, 1321122 - dir_dim // 2)
    b += struct.pack("<3QI", 4, 0, 2, K) + struct.pack(f"<{len(refcount)}i", *refcount)
    dim2 = dir_dim * dir_dim
    dirs = np.full((P, 2, dim2), -1, np.int32)
    if entries is None:
        dirs[:, 0, 10] = 0 | HOT
        dirs[0, 1, 10] = 1 | OWN | flags_extra
    else:
        for (p, kind, e), v in entries.items():
            dirs[p, kind, e] = v
    b += dirs.tobytes()
    rng_, n = np.random.default_rng(1), len(refcount)   # the payloads of the listed slots (a K field beyond them makes the file short)
    b += rng_.integers(0, 2**32, size=n * 1024, dtype=np.uint32).tobytes() + rng_.integers(0, 2**32, size=n * 32, dtype=np.uint32).tobytes()
    return b + trailing


def slam_payload(lidar=False, engine=False):
    b = struct.pack("<6d", 0.5, 0.5, 1.0 if lidar else 0.5, 0.0, 0.0, 0.05) + struct.pack("<IIii", 32, 100, 0, 1 if lidar else 0)
    b += bytes([1 if lidar else 0, 1 if lidar else 0]) + struct.pack("<iii", 64, 0, 2048)
    b += SE2_ID * 3 + b"\x00\x00" + struct.pack("<IQQ", 0, 0, 0) + struct.pack("<6Q", *([0] * 6)) * 2
    return b + b"\x00"


def _load(api, fn, path, dev=None):
    h = C.c_void_p()
    rc = fn(str(path).encode(), C.byref(dev) if dev is not None else None, C.byref(h))
    return rc, h


def _expect_valid(api, path, kind="pf"):
    L = api.lib()
    rc, h = _load(api, L.lama_pf_load_state if kind == "pf" else L.lama_slam_load_state, path)
    if api.device_count() < 1:
        assert rc == ERR_NO_DEVICE, (rc, L.lama_last_error())
        assert not h.value
    else:
        assert rc == OK, L.lama_last_error()
        (L.lama_pf_destroy if kind == "pf" else L.lama_slam_destroy)(h)


def _expect_bad(api, path, kind="pf", dev=None, msg=None):
    L = api.lib()
    rc, h = _load(api, L.lama_pf_load_state if kind == "pf" else L.lama_slam_load_state, path, dev)
    assert rc == ERR_ARG, (rc, L.lama_last_error())
    assert not h.value
    if msg:
        assert msg in L.lama_last_error().decode(), L.lama_last_error()


def test_python_written_file_is_read(api, tmp_path):
    # a filter after its first scan, one before it (no device state, no trajectory), a Slam2D and a LidarOdometry2D before their first scan
    for name, data, kind in [("pf", frame(pf_payload()), "pf"), ("pf_fresh", frame(pf_payload(engine=False, nodes=(), node_of=[-1] * 3)), "pf"),
                             ("slam", frame(slam_payload(), kind=2), "slam"), ("lo", frame(slam_payload(lidar=True), kind=3), "slam")]:
        p = tmp_path / f"{name}.ckpt"
        p.write_bytes(data)
        _expect_valid(api, p, kind)


@pytest.mark.parametrize("cut", [0, 7, 31, 33, 200, -4100, -1])
def test_truncated_files_are_refused(api, tmp_path, cut):
    data = frame(pf_payload())
    p = tmp_path / "t.ckpt"
    p.write_bytes(data[:cut] if cut >= 0 else data[:len(data) + cut])
    _expect_bad(api, p)


def test_header_corruptions_are_refused(api, tmp_path):
    data = bytearray(frame(pf_payload()))
    cases = {"magic": frame(pf_payload(), magic=b"LAMACKPX"), "version": frame(pf_payload(), version=2),
             "size": frame(pf_payload(), total=len(data) + 8), "checksum": frame(pf_payload(), checksum=12345)}
    flipped = bytearray(data)
    flipped[len(flipped) // 2] ^= 0x40
    cases["flipped payload byte"] = bytes(flipped)
    for name, b in cases.items():
        p = tmp_path / "h.ckpt"
        p.write_bytes(b)
        _expect_bad(api, p)


def test_wrong_kind_and_geometry_are_refused(api, tmp_path):
    p = tmp_path / "pf.ckpt"
    p.write_bytes(frame(pf_payload()))
    _expect_bad(api, p, kind="slam", msg="PFSlam2D")
    s = tmp_path / "slam.ckpt"
    s.write_bytes(frame(slam_payload(), kind=2))
    _expect_bad(api, s, kind="pf", msg="Slam2D")
    for field, v in [("dir_dim", 16), ("pool_slots", 17), ("max_beams", 1080)]:
        dev = api.DeviceOptions(device=0, dir_dim=0, pool_slots=0, max_beams=0, timing=0, stream=0)
        setattr(dev, field, v)
        _expect_bad(api, p, dev=dev, msg="geometry")
    dev = api.DeviceOptions(device=0, dir_dim=8, pool_slots=16, max_beams=2048, timing=0, stream=0)   # the saved values are accepted
    rc, h = _load(api, api.lib().lama_pf_load_state, p, dev)
    assert rc == (OK if api.device_count() else ERR_NO_DEVICE)
    api.lib().lama_pf_destroy(h)


@pytest.mark.parametrize("case", ["particles", "engine_particles", "slot_past_K", "flag_bits", "refcount", "node_order", "node_head", "rng",
                                  "trailing", "K_exceeds_file", "slam_in_pf_kind"])
def test_semantic_corruptions_with_a_valid_checksum_are_refused(api, tmp_path, case):
    kw = {"particles": dict(particles_field=1 << 30), "engine_particles": dict(engine_particles=4),
          "slot_past_K": dict(entries={(0, 0, 10): 2}, refcount=(1, 0)), "flag_bits": dict(flags_extra=1 << 27),
          "refcount": dict(refcount=(2, 1)), "node_order": dict(nodes=(1, -1)), "node_head": dict(node_of=[0, 0, 5]),
          "rng": dict(rng=b"1 2 3"), "trailing": dict(trailing=b"\x00"), "K_exceeds_file": dict(K=100000, pool=200000)}.get(case)
    p = tmp_path / "c.ckpt"
    p.write_bytes(frame(slam_payload(), kind=1) if case == "slam_in_pf_kind" else frame(pf_payload(**kw)))
    _expect_bad(api, p)


# ---- GPU: continuation == uninterrupted run ---------------------------------------------------------------------------------------
def _bytes(d):
    return {k: v.tobytes() for k, v in d.items()}


def _pf_maps(g, particles):
    out = []
    for p in particles:
        n0, mn0, mx0 = g.mapBounds(p, 0)
        n1, mn1, mx1 = g.mapBounds(p, 1)
        occ = _bytes(g.exportOccupancy(p, int(mn0[0]), int(mn0[1]), int(mx0[0] - mn0[0]), int(mx0[1] - mn0[1]))) if n0 else None
        dm = _bytes(g.exportDistance(p, int(mn1[0]), int(mn1[1]), int(mx1[0] - mn1[0]), int(mx1[1] - mn1[1]))) if n1 else None
        out.append((n0, mn0.tolist(), mx0.tolist(), n1, mn1.tolist(), mx1.tolist(), occ, dm))
    return out


def _counters(g):
    """the work counters without `detached`: how many copy-on-write copies a scan makes depends on which of the particles that share a
    patch reads its reference count first, so it differs between two uninterrupted runs (DESIGN.md §13).  A load restores it exactly."""
    return tuple({k: v for k, v in c.items() if k != "detached"} for c in g.counters())


def _pf_state(g, P, maps=None, traj=True):
    st, w = g.getParticles()
    d = dict(states=st.tobytes(), weights=w.tobytes(), neff=g.getNeff(), best=g.getBestParticleIdx(), last=g.lastResample().tolist(),
             digest=g.resampleDigest(), mem=g.getMemoryUsage(), stamps=g.getTimestamps(), counters=_counters(g))
    if traj:
        d["traj"] = [g.trajectory(i).tobytes() for i in range(P)]
    d["maps"] = _pf_maps(g, range(P) if maps is None else maps)
    return d


def _run_pf(api, ds, P, T, k, tmp_path, maps=None, traj_every=1, **opts):
    """A uninterrupted, S saved after scan k - 1 and continued, B loaded from S's file: all three equal after every scan"""
    mk = lambda: api.PFSlam2D(api.PFSlam2D.Options(P, trans_thresh=0.05, rot_thresh=0.05, seed=42, **opts))
    A, S = mk(), mk()
    for h in (A, S):
        h.setPrior(*ds.truth[0])
    B = None
    f1, f2 = tmp_path / "s.ckpt", tmp_path / "b.ckpt"
    for t in range(T):
        did = [h.update(ds.scans[t], ds.odom[t], timestamp=0.1 * t) for h in ([A, S] if B is None else [A, S, B])]
        assert len(set(did)) == 1, t
        if t == k - 1:
            S.saveState(f1)
            stats = api.checkpoint_stats()
            B = api.PFSlam2D.loadState(f1)
            assert B.summary() == S.summary() and B.getTimestamps() == S.getTimestamps() and B.counters() == S.counters()
            B.saveState(f2)                                              # canonical: save -> load -> save gives the same bytes
            assert f1.read_bytes() == f2.read_bytes()
            with pytest.raises(api.LamaError):                           # staged scans are not state
                B.updateStaged(0, ds.odom[t + 1])
        if t >= k - 1:
            full = (t - k) % traj_every == 0 or t == T - 1
            sa = _pf_state(A, P, maps if not full else None, traj=full)
            assert _pf_state(S, P, maps if not full else None, traj=full) == sa, t
            assert _pf_state(B, P, maps if not full else None, traj=full) == sa, t
    return stats, A


@pytest.mark.gpu
@pytest.mark.parametrize("gain", [None, 0.0008])
def test_pf_continuation_equals_uninterrupted_run(gpu_api, synth, tmp_path, gain):
    ds = synth.make_dataset("loop", 150, n_beams=1080)
    stats, A = _run_pf(gpu_api, ds, 32, 150, 75, tmp_path, **({} if gain is None else dict(meas_sigma_gain=gain)))
    assert stats["references"] > stats["used_slots"] > 0          # the save point falls where particles share patches
    assert stats["file_bytes"] == os.path.getsize(tmp_path / "s.ckpt")
    if gain is not None:
        assert A.resampleDigest()[0] >= 2


@pytest.mark.gpu
def test_pf_continuation_at_full_size(gpu_api, synth, tmp_path):
    """256 x 1080 with forced resampling: the production pool and a copy-out of several pinned chunks"""
    ds = synth.make_dataset("loop", 80, n_beams=1080)
    stats, A = _run_pf(gpu_api, ds, 256, 80, 40, tmp_path, maps=(0, 101, 255), traj_every=10, meas_sigma_gain=0.0008)
    assert stats["file_bytes"] > 2 * (8 << 20) and stats["references"] > stats["used_slots"]
    assert A.resampleDigest()[0] >= 1


def _near(scan, r):
    return np.ascontiguousarray(scan[np.hypot(scan[:, 0], scan[:, 1]) < r])


def _slam_state(g, logodds):
    d = dict(pose=g.getPose().tobytes(), state=g.state().tobytes(), cells=g.getNumberOfProcessedCells(), stats=g.mapStats(), counters=_counters(g))
    for kind in (0, 1):
        n, mn, mx = g.mapBounds(kind)
        d[f"bounds{kind}"] = (n, mn.tolist(), mx.tolist())
        if n:
            w, h = int(mx[0] - mn[0]), int(mx[1] - mn[1])
            if kind == 0:
                d["occ"] = _bytes(g.exportLogOdds(mn[0], mn[1], w, h) if logodds else g.exportOccupancy(mn[0], mn[1], w, h))
            else:
                d["dm"] = _bytes(g.exportDistance(mn[0], mn[1], w, h))
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["frequency", "logodds", "transient_map", "lidar_odometry"])
def test_slam_continuation_equals_uninterrupted_run(gpu_api, synth, tmp_path, mode):
    api = gpu_api
    ds = synth.make_dataset("corridor", 90, n_beams=720)
    if mode == "lidar_odometry":
        mk = lambda: api.LidarOdometry2D()
        step = lambda h, t: h.update(_near(ds.scans[t], 3.0))
    else:
        kw = dict(trans_thresh=0.05, rot_thresh=0.05, occupancy=int(mode == "logodds"), transient_map=int(mode == "transient_map"))
        mk = lambda: api.Slam2D(api.Slam2D.Options(**kw))
        scans = [(_near(s, 1.5) if mode == "transient_map" else s) for s in ds.scans]
        step = lambda h, t: h.update(scans[t], ds.odom[t])
    logodds = mode in ("logodds", "lidar_odometry")
    A, S = mk(), mk()
    if mode != "lidar_odometry":
        for h in (A, S):
            h.setPose(*ds.truth[0])
    B, k = None, 45
    for t in range(90):
        did = [step(h, t) for h in ([A, S] if B is None else [A, S, B])]
        assert len(set(did)) == 1, t
        if t == k - 1:
            S.saveState(tmp_path / "s.ckpt")
            B = api.Slam2D.loadState(tmp_path / "s.ckpt")
            assert isinstance(B, api.LidarOdometry2D) == (mode == "lidar_odometry") and B.counters() == S.counters()
        if B is not None:
            sa = _slam_state(A, logodds)
            assert _slam_state(S, logodds) == sa and _slam_state(B, logodds) == sa, t
    if mode == "transient_map" or mode == "lidar_odometry":
        assert A.mapStats()[1] > 0


@pytest.mark.gpu
def test_fresh_handles_twins_and_refusals(gpu_api, synth, tmp_path):
    """save before the first scan; two handles loaded from one file; a sharded handle is refused; corrupt real files give no handle"""
    api = gpu_api
    ds = synth.make_dataset("room", 24, n_beams=360)
    mk = lambda: api.PFSlam2D(api.PFSlam2D.Options(8, trans_thresh=0.05, rot_thresh=0.05, seed=9, meas_sigma_gain=0.002))
    A, F = mk(), mk()
    for h in (A, F):
        h.setPrior(*ds.truth[0])
    F.saveState(tmp_path / "fresh.ckpt")
    B = api.PFSlam2D.loadState(tmp_path / "fresh.ckpt")
    for t in range(12):
        assert A.update(ds.scans[t], ds.odom[t]) == B.update(ds.scans[t], ds.odom[t])
        assert _pf_state(A, 8) == _pf_state(B, 8), t
    A.saveState(tmp_path / "mid.ckpt")
    T1, T2 = api.PFSlam2D.loadState(tmp_path / "mid.ckpt"), api.PFSlam2D.loadState(tmp_path / "mid.ckpt")
    assert T1.counters() == T2.counters() == A.counters()
    for t in range(12, 24):
        assert len({h.update(ds.scans[t], ds.odom[t]) for h in (A, T1, T2)}) == 1
        sa = _pf_state(A, 8)
        assert _pf_state(T1, 8) == sa and _pf_state(T2, 8) == sa, t
    # Slam2D saved before its first scan
    sk = dict(trans_thresh=0.05, rot_thresh=0.05)
    SA, SF = api.Slam2D(api.Slam2D.Options(**sk)), api.Slam2D(api.Slam2D.Options(**sk))
    for h in (SA, SF):
        h.setPose(*ds.truth[0])
    SF.saveState(tmp_path / "slam_fresh.ckpt")
    SB = api.Slam2D.loadState(tmp_path / "slam_fresh.ckpt")
    for t in range(12):
        assert SA.update(ds.scans[t], ds.odom[t]) == SB.update(ds.scans[t], ds.odom[t])
        assert _slam_state(SA, False) == _slam_state(SB, False), t
    # a sharded handle cannot be saved
    sh = api.PFSlam2D(api.PFSlam2D.Options(8, shard_rank=0, shard_count=2, seed=3))
    with pytest.raises(api.LamaError) as e:
        sh.saveState(tmp_path / "sharded.ckpt")
    assert e.value.code == ERR_STATE
    # corrupt copies of a real file
    data = (tmp_path / "mid.ckpt").read_bytes()
    bad = tmp_path / "bad.ckpt"
    for cut in (16, 1000, len(data) // 2, len(data) - 1):
        bad.write_bytes(data[:cut])
        _expect_bad(api, bad)
    flipped = bytearray(data)
    flipped[len(data) - 5000] ^= 1
    bad.write_bytes(bytes(flipped))
    _expect_bad(api, bad, msg="checksum")
    bad.write_bytes(b"LAMACKPX" + data[8:])
    _expect_bad(api, bad)
    bad.write_bytes(data[:8] + struct.pack("<I", 9) + data[12:])
    _expect_bad(api, bad, msg="version")
    _expect_bad(api, tmp_path / "mid.ckpt", kind="slam")
    _expect_bad(api, tmp_path / "mid.ckpt", dev=api.DeviceOptions(device=0, dir_dim=32, pool_slots=0, max_beams=0, timing=0, stream=0))


SHIM_SRC = r'''
// a C++ caller through the shim: run, save, load, continue both, compare
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
int main(int argc, char** argv) {
  auto o = lama_b200_shim::PFSlam2D::defaults(8);
  o.seed = 11; o.trans_thresh = 0.05; o.rot_thresh = 0.05;
  lama_b200_shim::PFSlam2D a(o);
  a.setPrior(Pose{0, 0, 0});
  for (int t = 0; t < 6; ++t) a.update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0);
  a.saveState(argv[1]);
  auto b = lama_b200_shim::PFSlam2D::loadState(argv[1]);
  for (int t = 6; t < 12; ++t) {
    if (a.update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0) != b->update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0)) return 3;
    double pa[3], pb[3];
    a.getPose(pa); b->getPose(pb);
    if (pa[0] != pb[0] || pa[1] != pb[1] || pa[2] != pb[2] || a.getNeff() != b->getNeff()) return 4;
  }
  auto so = lama_b200_shim::Slam2D::defaults();
  so.trans_thresh = 0.05; so.rot_thresh = 0.05;
  lama_b200_shim::Slam2D s(so);
  for (int t = 0; t < 6; ++t) s.update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0);
  s.saveState(argv[2]);
  auto r = lama_b200_shim::Slam2D::loadState(argv[2]);
  for (int t = 6; t < 12; ++t) {
    s.update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0); r->update(scan(0.1 * t), Pose{0.1 * t, 0, 0}, 0.0);
    double pa[3], pb[3];
    s.getPose(pa); r->getPose(pb);
    if (pa[0] != pb[0] || pa[1] != pb[1] || pa[2] != pb[2] || s.getNumberOfProcessedCells() != r->getNumberOfProcessedCells()) return 5;
  }
  std::printf("shim checkpoints ok\n");
  return 0;
}
'''


def _build_shim(tmp_path):
    src = tmp_path / "ckpt.cpp"
    src.write_text(SHIM_SRC)
    exe = tmp_path / "ckpt"
    lib_dir = os.path.join(ROOT, "iris_lama_b200")
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", lib_dir, "-llama_b200",
                           f"-Wl,-rpath,{lib_dir}"])
    return exe


def test_shim_checkpoint_caller_compiles(api, tmp_path):
    _build_shim(tmp_path)


@pytest.mark.gpu
def test_shim_caller_saves_and_loads(gpu_api, tmp_path):
    exe = _build_shim(tmp_path)
    out = subprocess.run([str(exe), str(tmp_path / "pf.ckpt"), str(tmp_path / "slam.ckpt")], capture_output=True, text=True)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "shim checkpoints ok" in out.stdout
