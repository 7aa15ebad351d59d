"""3-D occupancy maps: FrequencyOccupancyMap / ProbabilisticOccupancyMap with is3d = true (src/sdm/*_occupancy_map.cpp, src/sdm/map.cpp).
CPU: the oracle (tests/occ3d_oracle.py) against hand cases, the device core (om3d_core.h) against the oracle bit for bit, the C-ABI,
the shim and .sdm parsing.  GPU: the device map (om3d.cu, lama_om3_*) against the oracle: cells, known bits, bounds, patch counts,
update counts, `changed` flags, queries, .sdm files and z-slice images."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

import occ3d_oracle as T

O = T.OFFSET
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ("frequency", "logodds")


def _logods(p):
    """logods() of probabilistic_occupancy_map.cpp:43-46: float in, double arithmetic, float out"""
    q = float(F(p))
    return F(math.log(q / (1.0 - q)))


def _box(m):
    n, mn, mx = m.bounds()
    return n, mn.copy(), (mx - mn).astype(np.int32)


def _same_cells(a, b, lo, size):
    ea, eb = a.export(lo, size), b.export(lo, size)
    assert np.array_equal(ea["known"], eb["known"])
    assert np.array_equal(ea["word"], eb["word"])
    return ea


def _random_clouds(rng, n, pts, spread=3.0):
    clouds = [rng.uniform(-spread, spread, (pts, 3)) for _ in range(n)]
    origins = [rng.uniform(-0.5, 0.5, 3) for _ in range(n)]
    quats = [np.r_[rng.normal(size=3) * 0.2, 1.0] for _ in range(n)]
    return clouds, np.array(origins), np.array([q / np.linalg.norm(q) for q in quats])


def _bresenham(a, b):
    """Map::computeRay (map.cpp:198-227), both ends excluded"""
    a, b = np.array(a, np.int64), np.array(b, np.int64)
    d = b - a
    step, d = np.where(d < 0, -1, 1), np.abs(d)
    n = int(d.max())
    err, c, out = np.zeros(3, np.int64), a.copy(), []
    for _ in range(n - 1):
        err += d
        for j in range(3):
            if 2 * err[j] >= n:
                c[j] += step[j]
                err[j] -= n
        out.append(tuple(int(x) for x in c))
    return out


# ---- CPU: the oracle on hand cases -----------------------------------------------------------------------------------------------
def test_oracle_axis_aligned_ray_excludes_both_ends():
    m = T.Oracle(0.1, "frequency")
    assert m.insertPointClouds([np.array([[1.0, 0.0, 0.0]])]) == 10          # the hit and 9 interior cells
    e = m.export(np.array([O, O, O], np.uint32), (16, 1, 1))
    row = e["word"][0, 0]
    assert e["known"][0, 0].tolist() == [0] + [1] * 10 + [0] * 5             # the sensor cell is not touched
    assert row[10] == 0x00010001 and all(row[c] == 0x00010000 for c in range(1, 10))


def test_oracle_three_axis_ray_cells():
    m = T.Oracle(0.1, "logodds")
    assert m.insertPointClouds([np.array([[0.52, -0.31, 0.24]])]) == 1 + 4
    ray = _bresenham((O, O, O), (O + 5, O - 3, O + 2))
    assert len(ray) == 4 and len({c[1] for c in ray}) > 1 and len({c[2] for c in ray}) > 1
    p, f = m.query(np.array(ray, np.uint32))
    assert (f == 1).all()                                                     # isFree, one miss each
    p, f = m.query(np.array([[O + 5, O - 3, O + 2], [O, O, O]], np.uint32))
    assert f.tolist() == [2, 4]


def test_oracle_logodds_saturates_at_both_clamps():
    m = T.Oracle(0.05, "logodds")
    c = np.array([[O + 3, O + 4, O + 5]], np.uint32)
    for _ in range(20):
        m.setOccupied(c)
    assert m.export(c[0], (1, 1, 1))["word"].view(F)[0, 0, 0] == _logods(0.97)
    for _ in range(40):
        m.setFree(c)
    assert m.export(c[0], (1, 1, 1))["word"].view(F)[0, 0, 0] == _logods(0.12)


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_set_unknown_return_values(kind):
    m = T.Oracle(0.05, kind)
    c = np.array([[O + 1, O + 2, O + 3]], np.uint32)
    assert not m.setUnknown(c)[0]                           # a fresh cell: visited 0 / log-odds 0 == occ_thresh_
    assert m.export(c[0], (1, 1, 1))["known"][0, 0, 0] == 1   # but Map::get allocated it and set its bit
    assert m.setOccupied(c)[0]
    assert m.setUnknown(c)[0]
    assert not m.setUnknown(c)[0]
    assert m.query(c)[1][0] == 4


def test_oracle_prune_resets_single_visits_and_keeps_the_known_bit():
    m = T.Oracle(0.05, "frequency")
    a, b, c = [np.array([[O + i, O, O]], np.uint32) for i in (1, 2, 3)]
    m.setOccupied(a)                  # {1, 1}: pruned
    m.setFree(b)                      # {0, 1}: pruned
    m.setFree(c), m.setFree(c)        # {0, 2}: kept
    m.prune()
    e = m.export(np.array([O + 1, O, O], np.uint32), (3, 1, 1))
    assert e["word"][0, 0].tolist() == [0, 0, 0x00020000] and e["known"][0, 0].tolist() == [1, 1, 1]


def test_oracle_update_order_changes_a_logodds_cell_at_the_clamp():
    """hit-then-miss and miss-then-hit differ at clamp_max: this is what the device's ordered fold must keep"""
    c = np.array([[O + 7, O + 7, O + 7]], np.uint32)
    out = []
    for ops in ([1, 0], [0, 1]):
        m = T.Oracle(0.05, "logodds")
        for _ in range(20):
            m.setOccupied(c)
        m.apply(np.repeat(c, 2, axis=0), ops)
        out.append(m.export(c[0], (1, 1, 1))["word"][0, 0, 0])
    assert out[0] != out[1]
    assert np.array([out[1]], np.uint32).view(F)[0] == _logods(0.97)


# ---- CPU: the device core against the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("full", [True, False])
def test_core_insertion_equals_oracle_bit_for_bit(kind, full):
    rng = np.random.default_rng(11)
    clouds, origins, quats = _random_clouds(rng, 6, 400)
    o, e = T.Oracle(0.05, kind), T.Emu(0.05, kind)
    assert o.insertPointClouds(clouds, origins, quats, full) == e.insertPointClouds(clouds, origins, quats, full)
    n, lo, size = _box(o)
    ex = _same_cells(o, e, lo, size)
    assert ex["known"].sum() > (5000 if full else 2000)
    q = np.c_[rng.integers(lo[0] - 40, lo[0] + size[0] + 40, 5000), rng.integers(lo[1] - 40, lo[1] + size[1] + 40, 5000),
              rng.integers(lo[2] - 40, lo[2] + size[2] + 40, 5000)].astype(np.uint32)
    (p1, f1), (p2, f2) = o.query(q), e.query(q)
    assert np.array_equal(p1, p2) and np.array_equal(f1, f2)
    if kind == "frequency":
        o.prune(), e.prune()
        _same_cells(o, e, lo, size)


@pytest.mark.parametrize("kind", KINDS)
def test_core_ordered_setters_equal_oracle(kind):
    rng = np.random.default_rng(4)
    cells = np.c_[O + rng.integers(-40, 40, (60, 3))].astype(np.uint32)
    pick = cells[rng.integers(0, len(cells), 20000)]
    ops = rng.choice([0, 1, 2], 20000, p=[0.45, 0.45, 0.1])
    o, e = T.Oracle(0.05, kind), T.Emu(0.05, kind)
    assert np.array_equal(o.apply(pick, ops), e.apply(pick, ops))
    _same_cells(o, e, np.array([O - 64] * 3, np.uint32), (128, 128, 128))


# ---- CPU: interface ------------------------------------------------------------------------------------------------------------
OM3 = ["lama_om3_create", "lama_om3_destroy", "lama_om3_insert_point_clouds", "lama_om3_apply", "lama_om3_query", "lama_om3_prune",
       "lama_om3_bounds", "lama_om3_export", "lama_om3_write", "lama_om3_read", "lama_om3_export_image", "lama_om3_kernel_times", "lama_w2m3"]


def test_new_symbols_declared_and_exported(api):
    src = open(os.path.join(ROOT, "include", "lama_b200.h")).read()
    L = api.lib()
    for n in OM3:
        assert re.search(r"\b%s\s*\(" % n, src) and n in api.EXPORTED_SYMBOLS and hasattr(L, n), n


def test_capi_null_handles_and_bad_arguments_are_refused(api):
    L = api.lib()
    null = C.c_void_p(None)
    u3 = (C.c_uint32 * 3)()
    i3 = (C.c_int32 * 3)(1, 1, 1)
    d2 = (C.c_int * 2)()
    calls = [
        (L.lama_om3_create, (C.c_double(0.05), C.c_uint32(32), C.c_int(0), null, null, null, null)),
        (L.lama_om3_insert_point_clouds, (null, null, null, C.c_int(0), null, null, C.c_int(1), null)),
        (L.lama_om3_apply, (null, null, null, C.c_int(0), null)),
        (L.lama_om3_query, (null, null, C.c_int(0), null, null)),
        (L.lama_om3_prune, (null,)),
        (L.lama_om3_bounds, (null, u3, u3, null)),
        (L.lama_om3_export, (null, u3, i3, null, null)),
        (L.lama_om3_write, (null, C.c_char_p(b"x.sdm"))),
        (L.lama_om3_read, (null, C.c_char_p(b"x.sdm"))),
        (L.lama_om3_export_image, (null, C.c_double(0), null, C.c_size_t(0), d2)),
        (L.lama_om3_kernel_times, (null, null, null)),
    ]
    for fn, args in calls:
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0
    assert L.lama_om3_destroy(null) == 0
    h = C.c_void_p()
    assert L.lama_om3_create(C.c_double(0.05), C.c_uint32(16), C.c_int(0), null, null, null, C.byref(h)) == -1   # patch_size != 32
    assert L.lama_om3_create(C.c_double(0.05), C.c_uint32(32), C.c_int(2), null, null, null, C.byref(h)) == -1   # no such kind
    big = (C.c_int32 * 3)(2048, 2048, 1)
    assert L.lama_om3_create(C.c_double(0.05), C.c_uint32(32), C.c_int(0), null, big, null, C.byref(h)) == -1    # > 65 536 entries


def test_w2m3_matches_the_oracle(api):
    rng = np.random.default_rng(2)
    p = rng.uniform(-50, 50, (1000, 3))
    assert np.array_equal(api.w2m3(0.05, p), T.w2m(0.05, p))


SHIM_SRC = r'''
#include <array>
#include <cstdio>
#include "lama_b200_shim.hpp"
struct Q { double x() const {return 0;} double y() const {return 0;} double z() const {return 0;} double w() const {return 1;} };
struct Cloud { std::vector<std::array<double,3>> points; std::array<double,3> sensor_origin_{}; Q sensor_orientation_; };
int main() {
  try {
    lama_b200_shim::OccupancyMap3D m(0.05, 1);
    auto c = std::make_shared<Cloud>(); c->points.push_back({1, 0.5, 0.25});
    std::printf("cells %llu\n", (unsigned long long)m.insertPointCloud(c));
    const uint32_t xyz[3] = {42275904u, 42275904u, 42275904u};
    std::printf("flags %d %d %d %f\n", (int)m.setOccupied(xyz), (int)m.isOccupied(xyz), (int)m.isUnknown(xyz), m.getProbability(xyz));
    m.setFree(xyz); m.setUnknown(xyz); m.write("/dev/null");
  } catch (const std::exception& e) { std::printf("%s\n", e.what()); }
  return 0; }
'''


def test_shim_occupancy3d_compiles_in_a_cpp_caller(api, tmp_path):
    src = tmp_path / "om3.cpp"
    src.write_text(SHIM_SRC)
    exe = tmp_path / "om3"
    lib_dir = os.path.join(ROOT, "iris_lama_b200")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", lib_dir, "-llama_b200",
                           f"-Wl,-rpath,{lib_dir}"])
    out = subprocess.check_output([str(exe)]).decode()
    if api.device_count() > 0:
        assert "cells 20" in out and "flags 1 1 0" in out, out
    else:
        assert out.startswith("lama_b200"), out                # loud failure without a GPU, never a CPU fallback


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_3d_sdm_file_parses(kind, tmp_path):
    from iris_lama_b200 import sdm
    rng = np.random.default_rng(8)
    clouds, origins, quats = _random_clouds(rng, 2, 200, 2.0)
    o = T.Oracle(0.1, kind)
    o.insertPointClouds(clouds, origins, quats)
    assert o.write(tmp_path / "o.sdm")
    f = sdm.read_sdm(tmp_path / "o.sdm")
    n, lo, size = _box(o)
    assert f["header"]["is_3d"] == 1 and f["header"]["cell_size"] == 4 and f["header"]["num_patches"] == n == len(f["patches"])
    assert f["header"]["resolution"] == F(0.1)
    for pid, (cells, mask) in f["patches"].items():
        x, y, z = sdm.patch_origin3(pid)
        assert cells.size == 32768 and mask.size == 512
        e = o.export(np.array([x, y, z], np.uint32), (32, 32, 32))
        assert np.array_equal(cells.view(np.uint32), e["word"].ravel())
        assert np.array_equal(np.unpackbits(mask.view(np.uint8), bitorder="little"), e["known"].ravel())


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _check_equal(g, o):
    ng, mng, mxg = g.bounds()
    no, mno, mxo = o.bounds()
    assert ng == no and np.array_equal(mng, mno) and np.array_equal(mxg, mxo)
    _, lo, size = _box(o)
    return _same_cells(g, o, lo, size)


def _check_queries(g, o, rng, n=20000):
    _, lo, size = _box(o)
    q = np.c_[rng.integers(lo[0] - 64, lo[0] + size[0] + 64, n), rng.integers(lo[1] - 64, lo[1] + size[1] + 64, n),
              rng.integers(lo[2] - 64, lo[2] + size[2] + 64, n)].astype(np.uint32)
    (pg, fg), (po, fo) = g.query(q), o.query(q)
    assert np.array_equal(fg, fo) and np.array_equal(pg.view(np.uint64), po.view(np.uint64))
    assert len(np.unique(fg)) >= 3


def _same_files(a, b):
    from iris_lama_b200 import sdm
    fa, fb = sdm.read_sdm(a), sdm.read_sdm(b)
    assert fa["header"].tobytes() == fb["header"].tobytes()
    assert fa["patches"].keys() == fb["patches"].keys()
    for k, (c, m) in fa["patches"].items():
        assert c.tobytes() == fb["patches"][k][0].tobytes() and np.array_equal(m, fb["patches"][k][1])


def _images(g, o):
    for zed in (-0.02, 0.4, 1.0, 1.9):
        a, b = g.exportImage(zed), o.exportImage(zed)
        assert a.shape == b.shape and np.array_equal(a, b), zed


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("res", [0.05, 0.1])
def test_gpu_lidar_clouds_equal_oracle(gpu_api, synth, kind, res, tmp_path):
    clouds, origins, quats = synth.make_clouds_3d(30 if res == 0.1 else 12)
    o = T.Oracle(res, kind)
    g = gpu_api.OccupancyMap3D(res, kind, center=(0, 0, 1.5))
    assert g.insertPointClouds(clouds, origins, quats) == o.insertPointClouds(clouds, origins, quats)
    ex = _check_equal(g, o)
    assert ex["known"].sum() > 100000
    _check_queries(g, o, np.random.default_rng(1))
    _images(g, o)
    g.write(tmp_path / "g.sdm")
    o.write(tmp_path / "o.sdm")
    _same_files(tmp_path / "g.sdm", tmp_path / "o.sdm")
    if kind == "frequency":
        g.prune(), o.prune()
        _check_equal(g, o)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_one_batch_over_several_sort_chunks_equals_per_cloud_calls_and_oracle(gpu_api, synth, kind):
    clouds, origins, quats = synth.make_clouds_3d(30)      # 864 000 points at 0.05 m: tens of millions of updates
    o = T.Oracle(0.05, kind)
    co = o.insertPointClouds(clouds, origins, quats)
    g1 = gpu_api.OccupancyMap3D(0.05, kind, center=(0, 0, 1.5))
    assert g1.insertPointClouds(clouds, origins, quats) == co
    g2 = gpu_api.OccupancyMap3D(0.05, kind, center=(0, 0, 1.5))
    assert sum(g2.insertPointClouds([c], origins[k:k + 1], quats[k:k + 1]) for k, c in enumerate(clouds)) == co
    assert co > 2 * (1 << 24)
    _check_equal(g1, o)
    _check_equal(g2, o)
    if kind == "logodds":
        _, launches = g1.kernelTimes()
        assert launches["insert"] >= 4 + 3 * 3            # mark, zero, scan, gather + (emit, sort, fold) per chunk


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_negative_coordinates_patch_boundaries_several_calls_full_on_and_off(gpu_api, kind):
    rng = np.random.default_rng(17)
    o = T.Oracle(0.05, kind)
    g = gpu_api.OccupancyMap3D(0.05, kind, window=(8, 8, 8))
    for call in range(4):
        clouds, origins, quats = _random_clouds(rng, 3, 3000, 3.0)    # world 0 is a patch corner: every axis crosses it
        full = call % 2 == 0
        assert g.insertPointClouds(clouds, origins, quats, full=full) == o.insertPointClouds(clouds, origins, quats, full=full)
    ex = _check_equal(g, o)
    assert ex["known"].sum() > 50000
    _check_queries(g, o, rng)
    _images(g, o)


@pytest.mark.gpu
def test_gpu_occupied_counter_wraps_without_touching_visited(gpu_api):
    cloud = [np.tile([[0.6, 0.35, -0.2]], (70000, 1))]           # 70 000 hits of one cell in one call
    o = T.Oracle(0.05, "frequency")
    g = gpu_api.OccupancyMap3D(0.05, "frequency")
    assert g.insertPointClouds(cloud) == o.insertPointClouds(cloud)
    ex = _check_equal(g, o)
    hit = T.w2m(0.05, cloud[0][:1])[0]
    _, lo, _ = _box(o)
    w = ex["word"][hit[2] - lo[2], hit[1] - lo[1], hit[0] - lo[0]]
    assert w == ((70000 - 65536) | ((70000 - 65536) << 16))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_apply_batch_with_repeated_cells_and_mixed_ops(gpu_api, kind):
    rng = np.random.default_rng(23)
    clouds, origins, quats = _random_clouds(rng, 2, 2000, 2.0)
    o = T.Oracle(0.05, kind)
    g = gpu_api.OccupancyMap3D(0.05, kind)
    g.insertPointClouds(clouds, origins, quats)
    o.insertPointClouds(clouds, origins, quats)
    cells = (O + rng.integers(-60, 60, (400, 3))).astype(np.uint32)    # some in patches the clouds never touched
    pick = cells[rng.integers(0, len(cells), 50000)]
    ops = rng.choice([0, 1, 2], 50000, p=[0.45, 0.45, 0.1])
    cg, co = g.apply(pick, ops), o.apply(pick, ops)
    assert np.array_equal(cg, co) and 100 < cg.sum() < len(cg)
    _check_equal(g, o)
    assert np.array_equal(g.setOccupied(cells[:50]), o.setOccupied(cells[:50]))
    assert np.array_equal(g.setUnknown(cells[:50]), o.setUnknown(cells[:50]))
    _check_equal(g, o)
    _check_queries(g, o, rng)


@pytest.mark.gpu
def test_gpu_window_and_pool_overflow_leave_the_map_unchanged(gpu_api):
    rng = np.random.default_rng(3)
    near, o1, q1 = _random_clouds(rng, 1, 500, 0.7)
    g = gpu_api.OccupancyMap3D(0.05, "logodds", window=(4, 4, 4))     # 6.4 m
    g.insertPointClouds(near, o1 * 0, q1)
    n0, lo, size = _box(g)
    before = g.export(lo, size)
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertPointClouds([np.array([[0.1, 0.1, 0.1], [5.0, 0.0, 0.0]])])
    assert e.value.code == -4
    with pytest.raises(gpu_api.LamaError) as e:
        g.apply(np.array([[O, O, O], [O + 200, O, O]], np.uint32), [1, 1])
    assert e.value.code == -4
    assert g.bounds()[0] == n0 and all(np.array_equal(before[k], g.export(lo, size)[k]) for k in before)

    p = gpu_api.OccupancyMap3D(0.05, "frequency", window=(4, 4, 4), pool_slots=n0)
    p.insertPointClouds(near, o1 * 0, q1)
    before = p.export(lo, size)
    with pytest.raises(gpu_api.LamaError) as e:
        p.insertPointClouds([np.array([[-2.0, -2.0, -2.0]])])        # inside the window, in patches the pool cannot hold
    assert e.value.code == -5
    assert p.bounds()[0] == n0 and all(np.array_equal(before[k], p.export(lo, size)[k]) for k in before)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_read_of_written_and_oracle_files(gpu_api, kind, tmp_path):
    rng = np.random.default_rng(9)
    clouds, origins, quats = _random_clouds(rng, 3, 1500, 2.0)
    o = T.Oracle(0.05, kind)
    g = gpu_api.OccupancyMap3D(0.05, kind)
    g.insertPointClouds(clouds, origins, quats)
    o.insertPointClouds(clouds, origins, quats)
    g.write(tmp_path / "g.sdm")
    o.write(tmp_path / "o.sdm")
    for path in ("g.sdm", "o.sdm"):
        r = gpu_api.OccupancyMap3D(0.05, kind)
        r.read(tmp_path / path)
        _check_equal(r, o)
        _check_queries(r, o, rng, 5000)
        r.write(tmp_path / ("r" + path))
        _same_files(tmp_path / ("r" + path), tmp_path / "o.sdm")
    with pytest.raises(gpu_api.LamaError):
        g.read(tmp_path / "o.sdm")                          # not empty
