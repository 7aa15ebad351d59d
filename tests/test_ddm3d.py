"""3-D DynamicDistanceMap: DynamicDistanceMap with is3d = true (src/sdm/dynamic_distance_map.cpp).
CPU: the oracle (tests/ddm3_oracle.py) against hand cases; the host build of the device core (ddm3_core.h) against the oracle bit for
bit on seeded add / remove stress, normally, under the stop-and-resume hooks and under ASan / UBSan; the host admission (window
margin, pool); the C-ABI's null checks and the shim.  GPU: the device map (ddm3d.cu, lama_dm3_*) against the oracle: every cell,
processed, bounds and patch sets after every update, the lidar scene with moving obstacles, the hooks, distance queries, .sdm files,
z-slice images and refusals."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ddm3_oracle as T

O = T.OFFSET
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REACHES = (1, 2, 10, 31, 63)
RESOLUTIONS = (0.05, 0.1)
HOOKS = {"LAMA_DM3_HEAP_CAP": "8", "LAMA_DM3_POP_BUDGET": "7"}


def _l2(reach, res):
    """an l2_max whose ceil(l2_max / res) is `reach`"""
    return (reach - 0.5) * res


def _window(reach):
    return (8, 8, 8) if reach > 20 else (8, 8, 4)


def _inner(reach, window):
    """the cells an admitted batch may hold: at least reach + 1 inside the window (centred on the origin) on every axis"""
    lo = np.array([O - 32 * (w // 2) for w in window], np.int64) + reach + 1
    hi = np.array([O - 32 * (w // 2) + 32 * w for w in window], np.int64) - 1 - (reach + 1)
    return lo, hi


def _cluster(rng, n, lo, hi, spread):
    c = rng.integers(lo, hi + 1)
    pts = np.rint(c + rng.normal(0, spread, (n, 3))).astype(np.int64)
    return np.clip(pts, lo, hi).astype(np.uint32)


def stress_steps(seed, reach):
    """seeded clustered add / remove batches, interleaved, with an update after some of them"""
    rng = np.random.default_rng(seed)
    window = _window(reach)
    lo, hi = _inner(reach, window)
    per = {1: 300, 2: 200, 10: 60, 31: 12, 63: 4}[reach]
    spread = max(2.0, reach / 2)
    present, steps = [], []
    for r in range(4 if reach < 31 else 2):
        new = np.concatenate([_cluster(rng, per, lo, hi, spread) for _ in range(2)])
        if present:
            old = np.array(present, np.uint32)
            gone = old[rng.random(len(old)) < 0.5]
            steps.append(("remove", np.concatenate([gone, new[:3]])))   # the last three are no-ops unless already obstacles
            present = [tuple(p) for p in old if tuple(p) not in {tuple(g) for g in gone}]
        steps.append(("add", np.concatenate([new, new[:5]])))           # repeated adds return early
        if r % 2 == 1:
            steps.append(("update",))
            steps.append(("add", _cluster(rng, per // 2 + 1, lo, hi, spread)))
        present += [tuple(p) for p in new]
        steps.append(("update",))
    return steps, window


def _run_check(tmp_path, steps, res, reach, window, sanitize, env=None, pool=0):
    scen = tmp_path / "scenario.bin"
    scen.write_bytes(T.scenario_bytes(steps))
    e = dict(os.environ, **(env or {}))
    if sanitize:
        e["ASAN_OPTIONS"] = "detect_leaks=1:abort_on_error=0"
        e["UBSAN_OPTIONS"] = "print_stacktrace=1:halt_on_error=1"
    r = subprocess.run([T.check_binary(sanitize), str(scen), repr(res), repr(_l2(reach, res)), *[str(w) for w in window], str(pool)], env=e,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok:" in r.stdout and "runtime error" not in r.stderr, r.stderr


def lidar_cells(res, n_clouds=30, step=1):
    """the distinct hit voxels (Map::w2m of every world point) of the synthetic 30-cloud lidar scene"""
    from iris_lama_b200 import synth
    clouds, origins, quats = synth.make_clouds_3d(n_clouds)
    pts = np.concatenate([c[::step] @ synth.quat_matrix(q).T + o for c, o, q in zip(clouds, origins, quats)])
    return np.unique(((pts * (1.0 / res) + float(O)) + 0.5).astype(np.uint32), axis=0)   # Map::w2m


# ---- CPU: the oracle on hand cases -------------------------------------------------------------------------------------------
def test_oracle_one_obstacle_exact_distances_and_offsets():
    reach, res = 4, 0.1
    m = T.Oracle(res, _l2(reach, res))
    assert m.max_sqdist == 16
    c = np.array([O + 10, O + 20, O + 30], np.uint32)
    m.addObstacle(c)
    m.update()
    lo = c - reach
    e = m.export(lo, (2 * reach + 1,) * 3)
    w = e["word"].astype(np.uint64)
    b = w.view(np.uint8).reshape(w.shape + (8,))
    for z in range(2 * reach + 1):
        for y in range(2 * reach + 1):
            for x in range(2 * reach + 1):
                d = np.array([x, y, z]) - reach
                sq = int(d @ d)
                cell = (z, y, x)
                if sq < 16:
                    assert e["known"][cell] and b[cell][3] & 1, d
                    assert int(w[cell] >> np.uint64(32)) == sq
                    assert [int(np.int8(v)) for v in b[cell][:3]] == list(-d)   # offset to the obstacle
                else:
                    assert not (b[cell][3] & 1)


def test_oracle_remove_leaves_touched_cells_invalid_and_known():
    reach, res = 3, 0.1
    m = T.Oracle(res, _l2(reach, res))
    c = np.array([O, O, O], np.uint32)
    m.addObstacle(c)
    m.update()
    e0 = m.export(c - reach - 1, (2 * reach + 3,) * 3)
    m.removeObstacle(c)
    m.update()
    e1 = m.export(c - reach - 1, (2 * reach + 3,) * 3)
    assert (e1["known"] >= e0["known"]).all() and e0["known"].sum() > 0
    touched = e1["known"] == 1
    assert (e1["word"][touched] == np.uint64(4 << 24)).all()   # known, invalid, not queued, offset 0, sqdist 0


def test_oracle_processed_counts():
    m = T.Oracle(0.1, _l2(1, 0.1))                 # max_sqdist 1: only the obstacle itself
    m.addObstacle(np.array([[O, O, O]], np.uint32))
    assert m.update() == 1
    m = T.Oracle(0.1, _l2(2, 0.1))                 # max_sqdist 4: the obstacle, 6 at sqdist 1, 12 at 2 and 8 at 3, each popped once
    m.addObstacle(np.array([[O, O, O]], np.uint32))
    assert m.update() == 1 + 6 + 12 + 8
    m.removeObstacle(np.array([[O, O, O]], np.uint32))
    assert m.update() == 1 + 6 + 12 + 8             # the raise wave pops every formerly valid cell
    assert m.update() == 0


def test_oracle_tie_follows_the_neighbour_order():
    """cells at equal distance from two obstacles keep the one whose wave reaches them first; the waves advance in the heap order of
    the pushes, which follow the neighbour order +x, +y, -x, -y, +z, -z"""
    m = T.Oracle(0.1, _l2(3, 0.1))
    a, b = np.array([O, O, O], np.uint32), np.array([O + 2, O + 2, O + 2], np.uint32)
    m.addObstacle(np.stack([a, b]))
    m.update()
    e = m.export(a, (3, 3, 3))
    w = e["word"].astype(np.uint64)
    off = w.view(np.uint8).reshape(w.shape + (8,))[..., :3].view(np.int8).astype(int)
    # (1, 1, 1) is at sqdist 3 from both: claimed by a (added first, popped first); (2, 1, 1) is 1 + 1 + 1 from a and 0 + 1 + 1 from b
    assert off[1, 1, 1].tolist() == [-1, -1, -1]
    assert off[1, 1, 2].tolist() == [0, 1, 1]
    # (0, 1, 1) and (1, 0, 1) tie at sqdist 2 from a only, (2, 2, 1) at 1 from b
    assert off[1, 2, 2].tolist() == [0, 0, 1]


def test_oracle_trilinear_distance_hand_and_finite_difference():
    res, reach = 0.1, 5
    m = T.Oracle(res, _l2(reach, res))
    m.addObstacle(np.array([[O + 3, O - 2, O + 1]], np.uint32))
    m.update()
    p = np.array([[0.123, -0.071, 0.044]])
    d, g = m.distance(p)
    mc = p[0] / res + O
    c = np.floor(mc).astype(np.int64)
    mu = mc - c
    vals = {}
    for i in range(8):
        k = np.array([i & 1, (i >> 1) & 1, i >> 2])
        vals[i] = m.cellDistance((c + k).astype(np.uint32)[None])[0]
        dd = (c + k) - np.array([O + 3, O - 2, O + 1])
        assert vals[i] == pytest.approx(np.sqrt(dd @ dd) * res)
    w = lambda i: np.prod([mu[j] if (i >> j) & 1 else 1 - mu[j] for j in range(3)])
    assert d[0] == pytest.approx(sum(vals[i] * w(i) for i in range(8)), abs=1e-12)
    h = 1e-3   # 0.01 cells: within the cell, where the interpolation is linear per axis; w2m's offset quantises finer steps
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        fd = (m.distance(p + e)[0][0] - m.distance(p - e)[0][0]) / (2 * h)
        assert g[0, k] == pytest.approx(fd, rel=1e-5, abs=1e-6)


def test_oracle_cell_distance_of_absent_and_invalid_cells():
    m = T.Oracle(0.05, 0.5)
    assert m.maxDistance() == pytest.approx(0.5)
    assert m.cellDistance(np.array([[O, O, O]], np.uint32))[0] == np.sqrt(100) * 0.05


# ---- CPU: the core against the oracle ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", RESOLUTIONS)
@pytest.mark.parametrize("reach", REACHES)
@pytest.mark.parametrize("hooks", (False, True), ids=("plain", "hooks"))
def test_core_matches_oracle_on_stress(tmp_path, reach, res, hooks):
    steps, window = stress_steps(100 + reach, reach)
    _run_check(tmp_path, steps, res, reach, window, sanitize=False, env=HOOKS if hooks else None)


@pytest.mark.parametrize("reach", (1, 10, 31))
def test_core_matches_oracle_under_sanitizers(tmp_path, reach):
    steps, window = stress_steps(200 + reach, reach)
    _run_check(tmp_path, steps, 0.1, reach, window, sanitize=True)
    _run_check(tmp_path, steps, 0.05, reach, window, sanitize=True, env=HOOKS)


def test_core_matches_oracle_on_lidar_obstacles(tmp_path):
    cells = lidar_cells(0.1, n_clouds=3, step=7)
    rng = np.random.default_rng(3)
    steps = [("add", cells), ("update",)]
    for _ in range(3):
        gone = cells[rng.random(len(cells)) < 0.05]
        steps += [("remove", gone), ("add", gone[::2] + np.array([1, 0, 0], np.uint32)), ("update",)]
    _run_check(tmp_path, steps, 0.1, 5, (8, 8, 4), sanitize=False)
    _run_check(tmp_path, steps, 0.1, 5, (8, 8, 4), sanitize=False, env=HOOKS)
    _run_check(tmp_path, steps[:2], 0.1, 5, (8, 8, 4), sanitize=True, env=HOOKS)


def test_core_hooks_resume_many_times(monkeypatch):
    for k, v in HOOKS.items():
        monkeypatch.setenv(k, v)
    e = T.Emu(0.1, _l2(10, 0.1))
    o = T.Oracle(0.1, _l2(10, 0.1))
    c = np.array([[O, O, O], [O + 7, O - 3, O + 2]], np.uint32)
    assert e.addObstacle(c) == 0
    o.addObstacle(c)
    assert e.update() == o.update()
    s = e.stats()
    assert s["launches"] > 500 and s["grows"] > 4 and s["lower_cap"] > 8
    T.same_maps(o, e)


# ---- CPU: the host admission -------------------------------------------------------------------------------------------------
def test_admission_refuses_cells_inside_the_margin_and_leaves_the_map_unchanged():
    reach = 10
    e = T.Emu(0.1, _l2(reach, 0.1), window=(8, 8, 4))
    lo, hi = _inner(reach, (8, 8, 4))
    ok = np.array([lo, hi], np.uint32)
    assert e.addObstacle(ok) == 0
    assert e.update() > 0
    before = e.patch_ids()
    for k in range(3):
        step = np.zeros(3, np.int64)
        step[k] = 1
        for bad in (lo - step, hi + step):
            assert e.addObstacle(np.stack([lo, bad]).astype(np.uint32)) == -4
            assert e.removeObstacle(np.stack([bad]).astype(np.uint32)) == -4
    assert e.update() == 0 and e.patch_ids() == before


def test_admission_refuses_batches_that_could_exhaust_the_pool():
    reach = 10
    e = T.Emu(0.1, _l2(reach, 0.1), window=(8, 8, 4), pool_slots=8)
    c = np.array([[O + 16, O + 16, O + 16]], np.uint32)   # the middle of a patch: reach 10 stays inside it
    assert e.addObstacle(c) == 0
    far = np.array([[O - 64, O - 64, O - 40]], np.uint32)   # a corner: 8 patches reachable, 7 more than there are free slots
    assert e.addObstacle(far) == -5
    assert e.update() > 0
    assert len(e.patch_ids()) == 1


# ---- CPU: C-ABI and shim -----------------------------------------------------------------------------------------------------
def test_capi_refuses_null_handles_and_outputs():
    from iris_lama_b200 import api
    L = api.lib()
    h = C.c_void_p()
    assert L.lama_dm3_create(C.c_double(0.1), C.c_uint32(32), C.c_double(0.5), None, None, None, None) == -1
    assert L.lama_dm3_create(C.c_double(0.1), C.c_uint32(16), C.c_double(0.5), None, None, None, C.byref(h)) == -1
    assert L.lama_dm3_create(C.c_double(0.01), C.c_uint32(32), C.c_double(1.0), None, None, None, C.byref(h)) == -1   # 100 cells
    for f, args in (("lama_dm3_max_sqdist", (None, None)), ("lama_dm3_max_distance", (None, None)), ("lama_dm3_add_obstacles", (None, None, 1)),
                    ("lama_dm3_remove_obstacles", (None, None, 1)), ("lama_dm3_update", (None, None)), ("lama_dm3_distance", (None, None, 1, None, None)),
                    ("lama_dm3_cell_distance", (None, None, 1, None)), ("lama_dm3_bounds", (None, None, None, None)),
                    ("lama_dm3_export", (None, None, None, None, None)), ("lama_dm3_write", (None, None)), ("lama_dm3_read", (None, None)),
                    ("lama_dm3_export_image", (None, C.c_double(0), None, C.c_size_t(0), None)), ("lama_dm3_kernel_times", (None, None, None)),
                    ("lama_dm3_run_stats", (None, None))):
        assert getattr(L, f)(*args) == -1, f
    assert L.lama_dm3_destroy(None) == 0


SHIM = r'''
#include <cstdio>
#include "lama_b200_shim.hpp"
int main() {
  try {
    lama_b200_shim::DynamicDistanceMap3D dm(0.1, 0.5);
    const uint32_t c[3] = {42275904u, 42275904u, 42275904u};
    dm.addObstacle(c); dm.removeObstacle(c);
    const double p[3] = {0, 0, 0}; double g[3];
    std::printf("processed %u %f %f %f\n", dm.update(), dm.distance(p, g), dm.distance(c), dm.maxDistance());
  } catch (const std::exception& e) { std::printf("%s\n", e.what()); }
  return 0; }
'''


def test_shim_compiles_and_links(tmp_path):
    src = tmp_path / "shim.cpp"
    src.write_text(SHIM)
    exe = tmp_path / "shim"
    lib_dir = os.path.join(ROOT, "iris_lama_b200")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", lib_dir, "-llama_b200",
                           f"-Wl,-rpath,{lib_dir}"])
    out = subprocess.check_output([str(exe)]).decode()
    assert "processed 2 " in out or "no CUDA device" in out or "device" in out


# ---- GPU: the device map against the oracle ----------------------------------------------------------------------------------
def _dev(res, reach, window=None, **kw):
    from iris_lama_b200 import api
    return api.DynamicDistanceMap3D(res, l2_max=_l2(reach, res), window=window, **kw)


def _dev_ids(m):
    """the device map's patches: the 32^3 blocks of its bounds with a known cell (Map::get marks the cell it allocates a patch for)"""
    n, mn, mx = m.bounds()
    ids = []
    for z in range(int(mn[2]), int(mx[2]) if n else 0, 32):
        for y in range(int(mn[1]), int(mx[1]), 32):
            for x in range(int(mn[0]), int(mx[0]), 32):
                if m.export(np.array([x, y, z], np.uint32), (32, 32, 32))["known"].any():
                    ids.append(((x >> 5) * T.UC + (y >> 5)) * T.UC + (z >> 5))
    assert len(ids) == n
    return sorted(ids)


def _same(o, m):
    T.same_maps(o, m, patch_ids=_dev_ids)


def _play(steps, o, m):
    for s in steps:
        if s[0] == "update":
            assert m.update() == o.update()
            _same(o, m)
        elif s[0] == "add":
            o.addObstacle(s[1])
            m.addObstacle(s[1])
        else:
            o.removeObstacle(s[1])
            m.removeObstacle(s[1])


@pytest.mark.gpu
@pytest.mark.parametrize("res", RESOLUTIONS)
@pytest.mark.parametrize("reach", REACHES)
def test_gpu_matches_oracle_on_stress(reach, res):
    steps, window = stress_steps(100 + reach, reach)
    o, m = T.Oracle(res, _l2(reach, res)), _dev(res, reach, window)
    _play(steps, o, m)
    assert m.max_sqdist == o.max_sqdist and m.maxDistance() == o.maxDistance()


@pytest.mark.gpu
def test_gpu_hooks_grow_heaps_and_resume(monkeypatch):
    for k, v in HOOKS.items():
        monkeypatch.setenv(k, v)
    steps, window = stress_steps(7, 10)
    o, m = T.Oracle(0.1, _l2(10, 0.1)), _dev(0.1, 10, window)
    _play(steps, o, m)
    s = m.runStats()
    assert s["launches"] > 500 and s["grows"] > 4


@pytest.mark.gpu
def test_gpu_lidar_scene_with_a_moving_box():
    res = 0.1
    cells = lidar_cells(res)
    o, m = T.Oracle(res, 0.5), _dev(res, 5)
    assert m.max_sqdist == 25
    o.addObstacle(cells)
    m.addObstacle(cells)
    assert m.update() == o.update()
    _same(o, m)
    box = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.uint32)
    at = np.array([O - 30, O - 20, O + 2], np.uint32)
    for r in range(20):
        nxt = at + np.array([3, 2, 0], np.uint32) if r % 4 != 3 else at - np.array([4, 1, 0], np.uint32)
        for mm in (o, m):
            if r:
                mm.removeObstacle(box + at)
            mm.addObstacle(box + nxt)
        assert m.update() == o.update(), r
        if r % 5 == 4:
            _same(o, m)
        at = nxt
    _same(o, m)


@pytest.mark.gpu
def test_gpu_distance_and_cell_distance_bit_equal():
    res = 0.05
    steps, _ = stress_steps(11, 10)
    o, m = T.Oracle(res, _l2(10, res)), _dev(res, 10)
    _play(steps, o, m)
    n, mn, mx = o.bounds()
    rng = np.random.default_rng(5)
    lo_w = (mn.astype(np.float64) - O - 5) * res
    hi_w = (mx.astype(np.float64) - O + 5) * res
    pts = rng.uniform(lo_w, hi_w, (100000, 3))
    pts[:1000] = np.round(pts[:1000] / res) * res              # on cell centres
    pts[1000:2000] = (mn.astype(np.float64) - O) * res           # on the bounds
    d0, g0 = o.distance(pts)
    d1, g1 = m.distance(pts)
    assert np.array_equal(d0, d1) and np.array_equal(g0, g1)
    assert np.array_equal(m.distance(pts, grad=False), d0)
    cells = rng.integers(mn.astype(np.int64) - 40, mx.astype(np.int64) + 40, (100000, 3)).astype(np.uint32)
    assert np.array_equal(o.cellDistance(cells), m.cellDistance(cells))


@pytest.mark.gpu
def test_gpu_sdm_files_and_images(tmp_path):
    res = 0.1
    steps, _ = stress_steps(13, 10)
    o, m = T.Oracle(res, _l2(10, res)), _dev(res, 10)
    _play(steps, o, m)
    o.write(tmp_path / "o.sdm")
    m.write(tmp_path / "m.sdm")
    ho, po, co = T.read_sdm(tmp_path / "o.sdm")
    hm, pm, cm = T.read_sdm(tmp_path / "m.sdm")
    assert ho == hm and po == pm and co == cm                    # bytes equal, patch order aside
    assert list(cm) == sorted(cm, key=lambda p: (p % T.UC, (p // T.UC) % T.UC, p // (T.UC * T.UC)))   # ascending window entry
    r = _dev(res, 10)
    r.read(tmp_path / "m.sdm")
    r.write(tmp_path / "r.sdm")
    assert (tmp_path / "r.sdm").read_bytes() == (tmp_path / "m.sdm").read_bytes()
    r2 = _dev(res, 10)
    r2.read(tmp_path / "o.sdm")
    _same(o, r2)
    for zed in (0.0, -0.4, 0.7, 2.0):
        assert np.array_equal(o.exportImage(zed), m.exportImage(zed))
    # the maps keep working after a read: the same batch on both
    extra = np.array([[O + 3, O + 1, O - 2]], np.uint32)
    o.addObstacle(extra)
    r2.addObstacle(extra)
    assert r2.update() == o.update()
    _same(o, r2)


def _corrupt(src, dst, fn):
    b = bytearray(open(src, "rb").read())
    fn(b)
    open(dst, "wb").write(bytes(b))


@pytest.mark.gpu
def test_gpu_refusals_leave_the_map_unchanged(tmp_path):
    from iris_lama_b200 import api
    res, reach = 0.1, 10
    o, m = T.Oracle(res, _l2(reach, res)), _dev(res, reach)
    c = np.array([[O, O, O]], np.uint32)
    o.addObstacle(c)
    m.addObstacle(c)
    m.update(), o.update()
    lo, hi = _inner(reach, (8, 8, 4))
    for bad in (lo - np.array([1, 0, 0]), hi + np.array([0, 0, 1])):
        with pytest.raises(api.LamaError) as ei:
            m.addObstacle(np.array([lo, bad], np.uint32))
        assert ei.value.code == -4
        with pytest.raises(api.LamaError) as ei:
            m.removeObstacle(np.array([bad], np.uint32))
        assert ei.value.code == -4
    assert m.update() == 0
    _same(o, m)
    small = _dev(res, reach, pool_slots=8)
    small.addObstacle(np.array([[O + 16, O + 16, O + 16]], np.uint32))
    with pytest.raises(api.LamaError) as ei:
        small.addObstacle(np.array([[O - 64, O - 64, O - 40]], np.uint32))
    assert ei.value.code == -5
    small.update()
    assert small.bounds()[0] == 1
    # files: a patch outside the window, a broken invariant, a reach above 63, an obstacle inside the margin
    m.write(tmp_path / "ok.sdm")
    hdr = 36

    def shift_id(b):
        pid = int(np.frombuffer(bytes(b[hdr:hdr + 8]), np.uint64)[0]) + 100 * T.UC * T.UC
        b[hdr:hdr + 8] = np.uint64(pid).tobytes()

    def bad_sqdist(b):
        cells = np.frombuffer(bytes(b[hdr + 8:hdr + 8 + 327680]), dtype=[("o", "<i2", 3), ("sq", "<u2"), ("v", "u1"), ("q", "u1")])
        k = hdr + 8 + 10 * int(np.nonzero(cells["v"] == 1)[0][0]) + 6   # sqdist of the first valid cell of the first patch
        b[k] += 1

    def big_reach(b):
        b[32:36] = np.uint32(64 * 64).tobytes()

    for name, fn, code in (("window", shift_id, -4), ("invariant", bad_sqdist, -1), ("reach", big_reach, -1)):
        _corrupt(tmp_path / "ok.sdm", tmp_path / f"{name}.sdm", fn)
        r = _dev(res, reach)
        with pytest.raises(api.LamaError) as ei:
            r.read(tmp_path / f"{name}.sdm")
        assert ei.value.code == code, name
        assert r.bounds()[0] == 0
        r.read(tmp_path / "ok.sdm")                    # still empty: the good file reads
        _same(o, r)
    edge = _dev(res, 2)
    edge.addObstacle(np.array([lo - 7], np.uint32))    # admitted with reach 2, inside the margin of reach 10
    edge.update()
    edge.write(tmp_path / "edge.sdm")
    _corrupt(tmp_path / "edge.sdm", tmp_path / "edge10.sdm", lambda b: b.__setitem__(slice(32, 36), np.uint32(100).tobytes()))
    r = _dev(res, reach)
    with pytest.raises(api.LamaError) as ei:
        r.read(tmp_path / "edge10.sdm")
    assert ei.value.code == -4 and r.bounds()[0] == 0
