"""The coupled 3-D map update: OccupancyMap3D.updateMaps / lama_om3_insert_point_clouds_dm3, the reference's map-update loop
(src/slam2d.cpp:271-316) with a 3-D occupancy map and a 3-D DynamicDistanceMap: `if (setOccupied(hit)) addObstacle(hit)`, along the
ray `if (setFree(c)) removeObstacle(c)`, update() after every cloud.
CPU: the host build of the per-cell filter and the segmented brushfire (tests/emu/occ_dist3_emu.cpp) against the oracle composition
(the occupancy oracle's setters, every one that returns true unfiltered through the distance oracle, tests/emu/occ_dist3_oracle.cpp) on seeded scenes, normally,
under the stop-and-resume hooks and under ASan / UBSan; the C-ABI's null checks; the shim.  GPU: the device maps against the oracle
composition (every occupancy and distance word, known bits, patch sets, bounds, processed per cloud, event and push counts,
trilinear distances) for both kinds, 0.1 and 0.05 m and reaches 1, 10 and 31; against the device's own ops (apply, add / remove,
update); refusals that leave both maps unchanged."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import ddm3_oracle as D

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(HERE, "emu")
O = D.OFFSET
UC = D.UC
KINDS = {"frequency": 0, "logodds": 1}
HOOKS = {"LAMA_DM3_HEAP_CAP": "8", "LAMA_DM3_POP_BUDGET": "7"}
CENTER = (0.0, 0.0, 1.5)
ORACLE_SRCS = [os.path.join(EMU, f) for f in ("occ_dist3_oracle.cpp", "occ3d_oracle.cpp", "ddm3_oracle.cpp")]


def _l2(reach, res):
    """an l2_max whose ceil(l2_max / res) is `reach`"""
    return (reach - 0.5) * res


def _window(res, reach):
    """the room (10 x 10 x 3 m) and the box path with the reach + 1 margin, centred on CENTER"""
    return (10, 10, 8) if res * (reach + 1) > 1.2 else (8, 8, 6)


# ---- fixtures: the oracle composition and the check binary ------------------------------------------------------------------
_lib = None
_check = {}


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def olib():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="occ_dist3_oracle_"), "libocc_dist3_oracle.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-ffp-contract=off", "-std=c++17", "-fPIC", "-Wall", "-shared", "-o", so, *ORACLE_SRCS])
        L = C.CDLL(so)
        L.o3o_create.restype = C.c_void_p
        L.o3o_create.argtypes = [C.c_double, C.c_int]
        L.d3o_create.restype = C.c_void_p
        L.d3o_create.argtypes = [C.c_double, C.c_double]
        L.od3o_update_maps.restype = C.c_uint64
        _lib = L
    return _lib


def check_binary(sanitize):
    """occ_dist3_check; with `sanitize` the host build (occ_dist3_emu.cpp) and the driver are built with -fsanitize=address,undefined and
    the oracles without (the oracle's ray code shifts negative error terms, which UBSan reports)"""
    if sanitize not in _check:
        d = tempfile.mkdtemp(prefix="occ_dist3_check_")
        exe = os.path.join(d, "occ_dist3_check")
        flags = ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"] if sanitize else ["-O2"]
        srcs = [os.path.join(EMU, "occ_dist3_check.cpp"), os.path.join(EMU, "occ_dist3_emu.cpp")]
        cxx = os.environ.get("CXX", "g++")
        compilers = [cxx, "g++", "/usr/bin/g++", "clang++"] if sanitize else [cxx]   # the first that links the sanitizer runtimes
        errors = []
        for c in dict.fromkeys(compilers):
            objs = [os.path.join(d, f"oracle{i}.o") for i in range(len(ORACLE_SRCS))]
            r = None
            for src, obj in zip(ORACLE_SRCS, objs):
                r = subprocess.run([c, "-std=c++17", "-ffp-contract=off", "-Wall", "-O2", "-c", "-o", obj, src], capture_output=True, text=True)
                if r.returncode != 0:
                    break
            if r.returncode == 0:
                r = subprocess.run([c, "-std=c++17", "-ffp-contract=off", "-Wall", *flags, "-o", exe, *srcs, *objs], capture_output=True, text=True)
            if r.returncode == 0:
                break
            errors.append(f"{c}: {r.stderr[-400:]}")
        else:
            raise RuntimeError("no compiler could build occ_dist3_check:\n" + "\n".join(errors))
        _check[sanitize] = exe
    return _check[sanitize]


class OracleMaps:
    """the reference's occupancy map and distance map, updated by the oracle composition"""

    def __init__(self, res, kind, reach, l2_max=None):
        L = olib()
        self.res, self.kind = res, kind
        self.om = C.c_void_p(L.o3o_create(res, KINDS[kind]))
        self.dm = C.c_void_p(L.d3o_create(res, _l2(reach, res) if l2_max is None else l2_max))

    def __del__(self):
        if _lib is not None and getattr(self, "om", None):
            _lib.o3o_destroy(self.om)
            _lib.d3o_destroy(self.dm)

    def addObstacle(self, cells):
        ops = D.ops_array(cells, 0)
        olib().d3o_apply(self.dm, _vp(ops), C.c_int(len(ops)))

    def updateMaps(self, clouds, origins=None, quats=None, full=True):
        p, off = _flat(clouds)
        o = None if origins is None else np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        q = None if quats is None else np.ascontiguousarray(quats, np.float64).reshape(-1, 4)
        processed, counts = np.zeros(len(off) - 1, np.uint32), np.zeros(2, np.uint64)
        n = olib().od3o_update_maps(self.om, self.dm, C.c_double(self.res), _vp(p), _vp(off), C.c_int(len(off) - 1), _vp(o), _vp(q), C.c_int(1 if full else 0),
                                    _vp(processed), _vp(counts))
        return int(n), processed, dict(events=int(counts[0]), pushes=int(counts[1]))

    def om_bounds(self):
        mn, mx = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        return olib().o3o_bounds(self.om, _vp(mn), _vp(mx)), mn, mx

    def om_export(self, lo, size=(32, 32, 32)):
        lo, sz = np.ascontiguousarray(lo, np.uint32), np.ascontiguousarray(size, np.int32)
        w, k = np.zeros(sz[::-1], np.uint32), np.zeros(sz[::-1], np.uint8)
        olib().o3o_export(self.om, _vp(lo), _vp(sz), _vp(w), _vp(k))
        return w, k

    def dm_view(self):
        return _DmView(self.dm)

    def distance(self, pts):
        p = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        d, g = np.zeros(len(p)), np.zeros((len(p), 3))
        olib().d3o_distance(self.dm, _vp(p), C.c_int(len(p)), _vp(d), _vp(g))
        return d, g


class _DmView:
    """the distance oracle as ddm3_oracle.same_maps reads a map"""

    def __init__(self, h):
        self.h = h

    def bounds(self):
        mn, mx = np.zeros(3, np.uint32), np.zeros(3, np.uint32)
        return olib().d3o_bounds(self.h, _vp(mn), _vp(mx)), mn, mx

    def patch_ids(self):
        n = self.bounds()[0]
        ids = np.zeros(max(n, 1), np.uint64)
        olib().d3o_patch_ids(self.h, _vp(ids))
        return sorted(int(i) for i in ids[:n])

    def export(self, lo, size):
        lo, sz = np.ascontiguousarray(lo, np.uint32), np.ascontiguousarray(size, np.int32)
        w, k = np.zeros(sz[::-1], np.uint64), np.zeros(sz[::-1], np.uint8)
        olib().d3o_export(self.h, _vp(lo), _vp(sz), _vp(w), _vp(k))
        return dict(word=w, known=k)


def _flat(clouds):
    clouds = [np.ascontiguousarray(c, np.float64).reshape(-1, 3) for c in clouds]
    off = np.zeros(len(clouds) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return np.ascontiguousarray(np.concatenate(clouds) if clouds else np.zeros((0, 3))), off


# ---- scenes --------------------------------------------------------------------------------------------------------------------
def box_points(center, size, n, rng):
    """n world points on the six faces of an axis-aligned box: rays to the far faces cross the near ones"""
    c, h = np.asarray(center, np.float64), np.asarray(size, np.float64) / 2
    u = rng.uniform(-1, 1, (n, 3))
    ax = rng.integers(0, 3, n)
    u[np.arange(n), ax] = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    return c + u * h


def scene_batches(n_batches, per_batch, step, seed, box_n=400):
    """[(clouds, origins, quats)] per batch: lidar clouds of synth.make_clouds_3d (every step-th point) interleaved with clouds of a 0.8 m
    box seen from two sensor positions; the box moves between batches and between the clouds of a batch, and returns to where it was,
    so cells turn occupied -> free -> occupied within a cloud, across the clouds of a batch and across batches"""
    from iris_lama_b200 import synth
    clouds, origins, quats = synth.make_clouds_3d(30)
    rng = np.random.default_rng(seed)
    ident = np.array([0.0, 0.0, 0.0, 1.0])
    out = []
    for b in range(n_batches):
        cs, os_, qs = [], [], []
        at = np.array([0.4 + 0.3 * b, -0.2 + 0.15 * b, 1.0])
        for j in range(per_batch):
            k = (b * per_batch + j) % 30
            cs.append(clouds[k][::step])
            os_.append(origins[k])
            qs.append(quats[k])
            if j % 2 == 0:
                where = at if j % 4 == 0 else at + np.array([0.25, 0.1, 0.0])
                eye = np.array([-1.5, -1.0, 1.2]) if j % 4 == 0 else np.array([1.8, 1.2, 0.8])
                cs.append(box_points(where, (0.8, 0.8, 0.8), box_n, rng) - eye)
                os_.append(eye)
                qs.append(ident)
        out.append((cs, np.array(os_), np.array(qs)))
    return out


def scenario_bytes(kind, res, reach, record_cap, window, batches, queued=None, dm_pool=0, full=True):
    """the scenario file of occ_dist3_check.cpp; queued[b] = cells added to the distance map before batch b"""
    v = [KINDS[kind], res, _l2(reach, res), record_cap, *window, dm_pool, 1 if full else 0, len(batches)]
    for b, (cs, os_, qs) in enumerate(batches):
        q = np.zeros((0, 3)) if not queued or b not in queued else np.asarray(queued[b], np.float64).reshape(-1, 3)
        v += [len(q), *q.ravel()]
        v.append(len(cs))
        for c, o, qq in zip(cs, os_, qs):
            v += [*o, *qq, len(c), *np.asarray(c, np.float64).ravel()]
    return np.asarray(v, "<f8").tobytes()


def centered_cells(res, pts):
    """Map::w2m of world points, as the maps compute it"""
    return ((np.asarray(pts, np.float64) * (1.0 / res) + float(O)) + 0.5).astype(np.uint32)


# ---- CPU: the host build against the oracle composition ------------------------------------------------------------------------
def _run_check(tmp_path, data, sanitize=False, env=None):
    scen = tmp_path / "scenario.bin"
    scen.write_bytes(data)
    e = dict(os.environ, **(env or {}))
    if sanitize:
        e["ASAN_OPTIONS"] = "detect_leaks=1:abort_on_error=0"
        e["UBSAN_OPTIONS"] = "print_stacktrace=1:halt_on_error=1"
    r = subprocess.run([check_binary(sanitize), str(scen)], env=e, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "ok:" in r.stdout and "runtime error" not in r.stderr, r.stderr
    return r.stdout


def _counts(out):
    ev = [int(l.split()[4]) for l in out.splitlines() if l.startswith("batch ")]
    push = [int(l.split()[6]) for l in out.splitlines() if l.startswith("batch ")]
    return ev, push


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("res,reach", [(0.1, 1), (0.1, 10), (0.05, 10), (0.1, 31)])
def test_core_matches_oracle_composition(tmp_path, kind, res, reach):
    batches = scene_batches(3, 4, 61, seed=reach)
    q = {1: centered_cells(res, [[0.5, 0.5, 0.5], [-1.0, 2.0, 1.0]])}   # queued addObstacles before the second call
    out = _run_check(tmp_path, scenario_bytes(kind, res, reach, 3000, _window(res, reach), batches, queued=q))
    ev, push = _counts(out)
    assert all(e > p > 0 for e, p in zip(ev, push)), (ev, push)   # the filter drops some events in every batch


def test_core_crosses_chunks_and_resumes_under_hooks(tmp_path):
    batches = scene_batches(2, 6, 97, seed=3)
    for kind in KINDS:
        data = scenario_bytes(kind, 0.1, 5, 700, _window(0.1, 5), batches, queued={0: centered_cells(0.1, [[0.0, 0.0, 1.0]])})
        _run_check(tmp_path, data)                 # chunks of at most 700 records: every batch crosses several
        _run_check(tmp_path, data, env=HOOKS)      # small heaps and pop budget: hundreds of stops and resumes


def test_core_without_rays(tmp_path):
    batches = scene_batches(2, 3, 101, seed=9)
    _run_check(tmp_path, scenario_bytes("logodds", 0.1, 10, 1 << 24, _window(0.1, 10), batches, full=False))


@pytest.mark.parametrize("reach", (1, 10))
def test_core_under_sanitizers(tmp_path, reach):
    batches = scene_batches(2, 3, 151, seed=20 + reach)
    _run_check(tmp_path, scenario_bytes("frequency", 0.1, reach, 500, _window(0.1, reach), batches), sanitize=True)
    _run_check(tmp_path, scenario_bytes("logodds", 0.05, reach, 500, _window(0.05, reach), batches), sanitize=True, env=HOOKS)


# ---- CPU: C-ABI and shim -----------------------------------------------------------------------------------------------------
def test_capi_refuses_null_handles():
    from iris_lama_b200 import api
    L = api.lib()
    f = L.lama_om3_insert_point_clouds_dm3
    off = np.zeros(2, np.int64)
    assert f(None, None, None, _vp(off), C.c_int(1), None, None, C.c_int(1), None, None, None) == -1
    assert f(None, None, None, None, C.c_int(0), None, None, C.c_int(1), None, None, None) == -1
    assert b"null" in L.lama_last_error()


SHIM = r'''
#include <array>
#include <cstdio>
#include "lama_b200_shim.hpp"
struct Q { double x() const {return 0;} double y() const {return 0;} double z() const {return 0;} double w() const {return 1;} };
struct Cloud { std::vector<std::array<double,3>> points; std::array<double,3> sensor_origin_{}; Q sensor_orientation_; };
int main() {
  try {
    lama_b200_shim::OccupancyMap3D om(0.1, 1);
    lama_b200_shim::DynamicDistanceMap3D dm(0.1, 0.25);
    auto c = std::make_shared<Cloud>(); c->points.push_back({1, 0.5, 0.25});
    std::printf("processed %u\n", om.updateMaps(dm, c));
  } catch (const std::exception& e) { std::printf("%s\n", e.what()); }
  return 0; }
'''


def test_shim_compiles_and_links(tmp_path):
    from iris_lama_b200 import api
    src = tmp_path / "shim.cpp"
    src.write_text(SHIM)
    exe = tmp_path / "shim"
    lib_dir = os.path.join(ROOT, "iris_lama_b200")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", lib_dir, "-llama_b200",
                           f"-Wl,-rpath,{lib_dir}"])
    out = subprocess.check_output([str(exe)]).decode()
    if api.device_count() > 0:
        assert out.startswith("processed ") and int(out.split()[1]) > 1, out   # the hit and the cells around it
    else:
        assert out.startswith("lama_b200"), out


# ---- GPU -----------------------------------------------------------------------------------------------------------------------
def _maps(res, kind, reach, window=None, **kw):
    from iris_lama_b200 import api
    window = window or _window(res, reach)
    om = api.OccupancyMap3D(res, kind, center=CENTER, window=window, **kw.get("om", {}))
    dm = api.DynamicDistanceMap3D(res, l2_max=_l2(reach, res), center=CENTER, window=window, **kw.get("dm", {}))
    return om, dm


def _blocks(m):
    """the allocated patches of a device map: the 32^3 blocks of its bounds with a known cell"""
    n, mn, mx = m.bounds()
    out = []
    for z in range(int(mn[2]), int(mx[2]) if n else 0, 32):
        for y in range(int(mn[1]), int(mx[1]), 32):
            for x in range(int(mn[0]), int(mx[0]), 32):
                e = m.export(np.array([x, y, z], np.uint32), (32, 32, 32))
                if e["known"].any():
                    out.append(((x >> 5) * UC + (y >> 5)) * UC + (z >> 5))
    assert len(out) == n
    return sorted(out)


def _same_om(o, om):
    ids = _blocks(om)
    n, mn, mx = o.om_bounds()
    gn, gmn, gmx = om.bounds()
    assert n == gn == len(ids) and np.array_equal(mn, gmn) and np.array_equal(mx, gmx)
    for pid in ids:
        lo = D.patch_anchor(pid)
        w, k = o.om_export(lo)
        e = om.export(lo, (32, 32, 32))
        assert np.array_equal(k, e["known"]), pid
        assert np.array_equal(w, e["word"]), pid


def _same(o, om, dm, rng=None):
    _same_om(o, om)
    D.same_maps(o.dm_view(), dm, patch_ids=_blocks)
    if rng is not None:   # trilinear distances and gradients, bit for bit
        n, mn, mx = o.dm_view().bounds()
        pts = rng.uniform((mn.astype(np.float64) - O) * o.res, (mx.astype(np.float64) - O) * o.res, (20000, 3))
        d0, g0 = o.distance(pts)
        d1, g1 = dm.distance(pts)
        assert np.array_equal(d0, d1) and np.array_equal(g0, g1)


def _play(batches, o, om, dm, queued=None, rng=None):
    totals = []
    for b, (cs, os_, qs) in enumerate(batches):
        if queued and b in queued:
            o.addObstacle(queued[b])
            dm.addObstacle(queued[b])
        n0, p0, c0 = o.updateMaps(cs, os_, qs)
        n1, p1, c1 = om.updateMaps(dm, cs, os_, qs, counts=True)
        assert n0 == n1 and c0 == c1, (b, c0, c1)
        assert np.array_equal(p0, p1), b
        _same(o, om, dm, rng)
        totals.append(c1)
    return totals


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("res", (0.1, 0.05))
@pytest.mark.parametrize("reach", (1, 10, 31))
def test_gpu_matches_oracle_composition(kind, res, reach):
    step = {1: 7, 10: 23, 31: 97}[reach] * (2 if res == 0.05 else 1)
    batches = scene_batches(3, 4, step, seed=reach)
    o, (om, dm) = OracleMaps(res, kind, reach), _maps(res, kind, reach)
    q = {1: centered_cells(res, [[0.5, 0.5, 0.5], [-1.0, 2.0, 1.0]])}
    totals = _play(batches, o, om, dm, queued=q, rng=np.random.default_rng(reach))
    assert all(t["events"] > t["pushes"] > 0 for t in totals), totals


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_thirty_clouds_at_5cm_cross_record_chunks(kind):
    """the whole 30-cloud lidar scene at 0.05 m in one call (tens of millions of records, so several sort chunks), then the box batch"""
    from iris_lama_b200 import synth
    clouds, origins, quats = synth.make_clouds_3d(30)
    res, reach = 0.05, 1
    o, (om, dm) = OracleMaps(res, kind, reach), _maps(res, kind, reach, om=dict(timing=1))
    n0, p0, c0 = o.updateMaps(clouds, origins, quats)
    n1, p1, c1 = om.updateMaps(dm, clouds, origins, quats, counts=True)
    assert n1 > 3 * (1 << 24)
    assert n0 == n1 and c0 == c1 and np.array_equal(p0, p1)
    assert om.kernelTimes()[1]["insert"] > 3 * 8   # the chunk loop ran more than three times
    _same(o, om, dm)
    _play(scene_batches(1, 4, 13, seed=1), o, om, dm)


_HOOK_SCRIPT = r'''
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import test_occ_dist3d as T
for kind in T.KINDS:
    o, (om, dm) = T.OracleMaps(0.1, kind, 10), T._maps(0.1, kind, 10)
    T._play(T.scene_batches(2, 4, 41, seed=4), o, om, dm, queued={{0: T.centered_cells(0.1, [[0.0, 0.0, 1.0]])}})
    s = dm.runStats()
    assert s["launches"] > 500 and s["grows"] > 4, s
print("hooks ok")
'''


@pytest.mark.gpu
def test_gpu_hooks_grow_heaps_and_resume():
    env = dict(os.environ, **HOOKS)
    r = subprocess.run([sys.executable, "-c", _HOOK_SCRIPT.format(root=ROOT, tests=HERE)], env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0 and "hooks ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def _ray(a, b):
    """Map::computeRay (the reference's 3-D Bresenham), both ends excluded"""
    a, b = [int(v) for v in a], [int(v) for v in b]
    d = [b[j] - a[j] for j in range(3)]
    step = [-1 if v < 0 else 1 for v in d]
    d = [abs(v) for v in d]
    n = max(d)
    err, c, out = [0, 0, 0], list(a), []
    for _ in range(n - 1):
        for j in range(3):
            err[j] += d[j]
        for j in range(3):
            if (err[j] << 1) >= n:
                c[j] += step[j]
                err[j] -= n
        out.append(tuple(c))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_equals_the_device_composition(kind):
    """a sensor at the world origin: the literal op list (hit, then the ray) through apply, its changed flags as add / remove, update()
    per cloud; the occupancy map also equals insertPointClouds"""
    from iris_lama_b200 import api
    rng = np.random.default_rng(11)
    res, reach = 0.1, 4
    clouds = [box_points((0.6 + 0.2 * k, -0.3, 1.0 + 0.1 * k), (0.8, 0.6, 0.5), 150, rng) for k in range(4)]
    om, dm = _maps(res, kind, reach)
    om2, dm2 = _maps(res, kind, reach)
    om3, _ = _maps(res, kind, reach)
    n, processed = om.updateMaps(dm, clouds)
    assert om3.insertPointClouds(clouds) == n
    so = centered_cells(res, [[0.0, 0.0, 0.0]])[0]
    expect = []
    for c in clouds:
        cells, ops = [], []
        for h in centered_cells(res, c):
            cells.append(h)
            ops.append(api.OccupancyMap3D.SET_OCCUPIED)
            for r in _ray(so, h):
                cells.append(r)
                ops.append(api.OccupancyMap3D.SET_FREE)
        cells, ops = np.array(cells, np.uint32), np.array(ops, np.uint8)
        changed = om2.apply(cells, ops)
        for cell, op in zip(cells[changed], ops[changed]):
            (dm2.addObstacle if op == api.OccupancyMap3D.SET_OCCUPIED else dm2.removeObstacle)(cell[None])
        expect.append(dm2.update())
    assert processed.tolist() == expect
    for a in (om2, om3):
        ids = _blocks(om)
        assert ids == _blocks(a)
        for pid in ids:
            lo = D.patch_anchor(pid)
            ea, eb = om.export(lo, (32, 32, 32)), a.export(lo, (32, 32, 32))
            assert np.array_equal(ea["word"], eb["word"]) and np.array_equal(ea["known"], eb["known"])
    ids = _blocks(dm)
    assert ids == _blocks(dm2)
    for pid in ids:
        lo = D.patch_anchor(pid)
        assert np.array_equal(dm.export(lo, (32, 32, 32))["word"], dm2.export(lo, (32, 32, 32))["word"])


def _snapshot(om, dm):
    out = []
    for m in (om, dm):
        n, mn, mx = m.bounds()
        out.append((n, mn.tolist(), mx.tolist(), [(pid, m.export(D.patch_anchor(pid), (32, 32, 32))["word"].tobytes(),
                                                    m.export(D.patch_anchor(pid), (32, 32, 32))["known"].tobytes()) for pid in _blocks(m)]))
    return out


@pytest.mark.gpu
def test_gpu_refusals_leave_both_maps_unchanged():
    from iris_lama_b200 import api
    res, reach = 0.1, 10
    batches = scene_batches(1, 2, 53, seed=2)
    cs, os_, qs = batches[0]

    # the window margin: the window (4 patches on z) spans z = -6.4 .. 6.3 m; a hit at z = 6.0 m is inside it but less than reach + 1
    # = 11 cells from its edge
    eye, ident = np.array([[0.0, 0.0, 1.5]]), np.array([[0, 0, 0, 1.0]])
    for kind in KINDS:
        om, dm = _maps(res, kind, reach, window=(4, 4, 4))
        om.updateMaps(dm, [np.array([[0.5, 0.5, 0.0]])], eye, ident)
        dm.addObstacle(centered_cells(res, [[0.2, 0.2, 1.0]]))           # queued: stays queued after the refusal
        before = _snapshot(om, dm)
        with pytest.raises(api.LamaError) as ei:
            om.updateMaps(dm, [np.array([[0.5, 0.5, 0.0]]), np.array([[0.5, 0.5, 4.5]])], np.repeat(eye, 2, 0), np.repeat(ident, 2, 0))
        assert ei.value.code == -4 and _snapshot(om, dm) == before
        om.updateMaps(dm, [np.array([[0.5, 0.5, 3.0]])], eye, ident)     # 4.5 m: admitted
    # each pool
    om, dm = _maps(res, "frequency", reach, om=dict(pool_slots=2))
    with pytest.raises(api.LamaError) as ei:
        om.updateMaps(dm, cs, os_, qs)
    assert ei.value.code == -5 and om.bounds()[0] == 0 and dm.bounds()[0] == 0
    om, dm = _maps(res, "frequency", reach, dm=dict(pool_slots=3))
    with pytest.raises(api.LamaError) as ei:
        om.updateMaps(dm, cs, os_, qs)
    assert ei.value.code == -5 and om.bounds()[0] == 0 and dm.bounds()[0] == 0
    # mismatched geometry: resolution, window, centre
    om, dm = _maps(res, "frequency", reach)
    om.updateMaps(dm, cs[:1], os_[:1], qs[:1])
    for other in (api.DynamicDistanceMap3D(0.05, l2_max=0.5, center=CENTER, window=_window(res, reach)),
                  api.DynamicDistanceMap3D(res, l2_max=_l2(reach, res), center=CENTER, window=(8, 8, 8)),
                  api.DynamicDistanceMap3D(res, l2_max=_l2(reach, res), center=(4.0, 0.0, 1.5), window=_window(res, reach))):
        before = _snapshot(om, other)
        with pytest.raises(api.LamaError) as ei:
            om.updateMaps(other, cs, os_, qs)
        assert ei.value.code == -1 and _snapshot(om, other) == before
