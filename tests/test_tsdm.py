"""TruncatedSignedDistanceMap (src/sdm/truncated_signed_distance_map.cpp), toMesh and sdm::export_to_ply.
CPU: the oracle (tests/tsdm_oracle.py) against hand cases, the device fusion core (tsdm_core.h) against the oracle bit for bit, the
generated marching-cubes table, meshes of an analytic sphere, the C-ABI boundary.  GPU: the device map (tsdm.cu, lama_tsdm_*) against
the oracle: cells, "on" bits, bounds, patch count, return values, distance queries, meshes and PLY files."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

import tsdm_oracle as T

O = T.OFFSET
F = np.float32


def _qz(theta):
    return np.array([0.0, 0.0, math.sin(theta / 2), math.cos(theta / 2)])


def _box(m, is3d):
    n, mn, mx = m.bounds()
    size = (mx - mn).astype(np.int32)
    lo = mn.copy()
    if not is3d:
        lo[2], size[2] = 0, 1
    return n, lo, size


def _bits_equal(a, b):
    """bit-for-bit equal floats, except that a NaN equals any NaN: a cell whose first fold has weight 0 (d == -delta_ exactly) holds
    0 / 0 in the reference too, and the host and the device make NaNs of different bit patterns"""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a).view(np.uint32), np.where(nb, 0, b).view(np.uint32))


def _same_cells(a, b, lo, size):
    ea, eb = a.export(lo, size), b.export(lo, size)
    assert np.array_equal(ea["on"], eb["on"])
    for k in ("distance", "weight"):
        assert _bits_equal(ea[k], eb[k]), k
    return ea


# ---- CPU: the oracle on hand cases -----------------------------------------------------------------------------------------------
def _expected_ray(res, hit_x, trunc, cells):
    """integrate((0,0,0), (hit_x,0,0)) restated in closed form for an axis-aligned ray: {cell x: (distance, weight) or None (skipped)}"""
    sq = F(hit_x * hit_x)
    inv_sq = F(1.0 / float(sq))
    delta, eps = F(4 * res), F(res)
    inv_de = F(1.0 / float(delta - eps))
    out = {}
    for c in cells:
        d = F(abs(hit_x - (c - O) * res) * np.sign(hit_x - (c - O) * res))
        if d < -delta:
            out[c] = None
        elif -delta <= d <= -eps:
            out[c] = (d, F(F(F(d + delta) * inv_sq) * inv_de))
        else:
            out[c] = (d, inv_sq)
    return out


def test_oracle_axis_ray_closed_form_on_both_sides_of_delta_and_epsilon():
    res = 0.05
    m = T.Oracle(res)
    m.setMaxDistance(0.5)                        # the far side reaches past -delta_ = -0.2: skipped voxels
    assert m.insertPointCloud(np.array([[2.0, 0.0, 0.0]])) == 1
    lo = np.array([O, O, 0], np.uint32)
    e = m.export(lo, (64, 1, 1))
    on = np.flatnonzero(e["on"][0, 0])
    # computeRay(w2m(2.0 - 0.5), w2m(2.0 + 0.5)) excludes both ends: cells 31..49
    assert on.tolist() == list(range(31, 50))
    exp = _expected_ray(res, 2.0, 0.5, [O + c for c in on])
    kinds = set()
    for c in on:
        x = exp[O + c]
        if x is None:                            # skipped: allocated, "on", weight 0
            assert e["weight"][0, 0, c] == 0 and e["distance"][0, 0, c] == 0
            kinds.add("skip")
        elif x[1] == 0:                          # d == -delta_ exactly: weight 0, and the fold divides 0 by 0 as the reference does
            assert e["weight"][0, 0, c] == 0 and np.isnan(e["distance"][0, 0, c])
            kinds.add("nan")
        else:                                    # first fold from {0, 0}: (0 * 0 + w d) / (0 + w)
            d, w = x
            assert e["weight"][0, 0, c] == w and e["distance"][0, 0, c] == F(F(w * d) / w)
            kinds.add("ramp" if w != F(1.0 / 4.0) else "flat")
    assert kinds == {"skip", "nan", "ramp", "flat"}


def test_oracle_near_point_truncates_with_the_squared_norm():
    """|hit| = 0.2 m: squared norm 0.04 < 0.15, so the walk starts 0.04 m (not 0.15 m) before the hit"""
    m = T.Oracle(0.01)
    m.insertPointCloud(np.array([[0.2, 0.0, 0.0]]))
    e = m.export(np.array([O, O, 0], np.uint32), (64, 1, 1))
    # start = w2m(0.16) = 16, end = w2m(0.35) = 35, both excluded
    assert np.flatnonzero(e["on"][0, 0]).tolist() == list(range(17, 35))


def test_oracle_two_points_in_one_hit_cell_integrate_once():
    a, b = T.Oracle(0.05), T.Oracle(0.05)
    assert a.insertPointCloud(np.array([[1.0, 0.5, 0.0], [1.01, 0.5, 0.0], [1.0, 1.5, 0.0]])) == 2
    b.insertPointCloud(np.array([[1.0, 0.5, 0.0], [1.0, 1.5, 0.0]]))
    n, lo, size = _box(a, False)
    _same_cells(a, b, lo, size)


def test_oracle_weight_clamps_at_maximum_weight():
    m = T.Oracle(0.05)
    cloud = np.array([[0.1, 0.0, 0.0]])          # inv_squared_norm = 100 per fold
    for _ in range(120):
        m.insertPointCloud(cloud)
    e = m.export(np.array([O, O, 0], np.uint32), (8, 1, 1))
    assert e["weight"].max() == F(10000)


def test_oracle_tilted_2d_ray_folds_one_cell_several_times():
    """in 2-D the walk still carries z: a steep ray visits one (x, y) cell at several z, one fold each"""
    m = T.Oracle(0.05)
    m.setMaxDistance(0.3)
    m.integrate([0, 0, 0], [0.5, 0.0, 2.0])
    sq = 0.5 ** 2 + 2.0 ** 2
    e = m.export(np.array([O, O, 0], np.uint32), (16, 1, 1))
    assert e["weight"].max() > F(1.0 / sq) * F(1.5)       # one fold weighs at most inv_squared_norm
    em = T.Emu(0.05)
    em.insertPointClouds([np.array([[0.5, 0.0, 2.0]])])
    o2 = T.Oracle(0.05)
    o2.insertPointCloud(np.array([[0.5, 0.0, 2.0]]))
    _same_cells(o2, em, np.array([O, O, 0], np.uint32), (16, 1, 1))


def test_oracle_unknown_cell_reads_truncate_size():
    m = T.Oracle(0.05)
    d, g = m.distance(np.array([[3.0, 3.0, 0.0]]), gradient=True)
    assert d[0] == F(0.15) and not g.any()
    m.setMaxDistance(0.3)
    assert m.distance(np.array([[3.0, 3.0, 0.0]]))[0] == F(0.3)


@pytest.mark.parametrize("is3d", [False, True])
def test_oracle_gradient_matches_finite_differences(is3d):
    res = 0.05
    m = T.Oracle(res, is3d)
    rng = np.random.default_rng(3)
    dirs = rng.normal(size=(2000, 3))
    if not is3d:
        dirs[:, 2] = 0
    dirs /= np.linalg.norm(dirs, axis=1)[:, None]
    m.insertPointCloud(dirs * 1.0)
    # points inside one cell interval on every axis (away from the cell boundaries), near the surface
    base = dirs[:200] * 1.0
    cells = np.floor(base / res + O) - O
    pts = (cells + 0.3 + 0.4 * rng.random(base.shape)) * res
    if not is3d:
        pts[:, 2] = 0
    d, g = m.distance(pts, gradient=True)
    h = 1e-3                                     # world -> map adds 42 275 904 cells: a smaller step drowns in its rounding
    for k in range(3 if is3d else 2):
        dp = np.zeros(3)
        dp[k] = h
        fd = (m.distance(pts + dp) - m.distance(pts - dp)) / (2 * h)
        assert np.allclose(g[:, k], fd, rtol=1e-4, atol=1e-5), k


# ---- CPU: the device fusion core against the oracle ------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["2d", "2d_tilted", "3d"])
def test_fusion_core_equals_oracle_bit_for_bit(case):
    rng = np.random.default_rng(11)
    is3d = case == "3d"
    o, e = T.Oracle(0.05, is3d), T.Emu(0.05, is3d)
    clouds, origins, quats = [], [], []
    for k in range(6):
        p = rng.uniform(-3, 3, (400, 3))
        if case == "2d":
            p[:, 2] = 0
        clouds.append(p)
        origins.append(rng.uniform(-0.5, 0.5, 3) * (1 if case != "2d" else np.array([1, 1, 0])))
        quats.append(np.r_[rng.normal(size=3) * (0.2 if case != "2d" else 0), 1.0])
    quats = [q / np.linalg.norm(q) for q in quats]
    assert np.array_equal(o.insertPointClouds(clouds, origins, quats), e.insertPointClouds(clouds, origins, quats))
    n, lo, size = _box(o, is3d)
    assert n > 0
    ex = _same_cells(o, e, lo, size)
    assert ex["on"].sum() > 1000
    q = rng.uniform(-3, 3, (2000, 3))
    d1, g1 = o.distance(q, True)
    d2, g2 = e.distance(q, True)
    assert np.array_equal(d1, d2) and np.array_equal(g1, g2)


def test_mesh_vertex_core_equals_oracle_on_a_3d_map():
    tri, _ = T.mc_table()
    o, e = T.Oracle(0.1, True), T.Emu(0.1, True)
    rng = np.random.default_rng(5)
    dirs = rng.normal(size=(3000, 3))
    dirs /= np.linalg.norm(dirs, axis=1)[:, None]
    for m in (o, e):
        m.insertPointCloud(dirs * 1.0)
    verts = o.toMesh()
    assert len(verts) > 30
    # the oracle's first cubes again through mc_cube + mc_edge_vertex
    n, lo, size = _box(o, True)
    ex = o.export(lo, size)
    got = []
    for z, y, x in zip(*np.nonzero(ex["on"])):
        cfg, v = e.cube((lo[0] + x, lo[1] + y, lo[2] + z), tri)
        if cfg > 0 and cfg < 255:
            got.append(v[:3 * int((tri[cfg] >= 0).sum() // 3)])
    got = np.concatenate(got)
    assert len(got) == len(verts)
    assert set(map(tuple, got.tolist())) == set(map(tuple, verts.tolist()))


# ---- CPU: the generated triangle table -------------------------------------------------------------------------------------------
CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGE = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
FACE = [(0, 1, 2, 3), (4, 5, 6, 7), (0, 1, 5, 4), (3, 2, 6, 7), (0, 3, 7, 4), (1, 2, 6, 5)]


def _edge_of(a, b):
    return next(i for i, e in enumerate(EDGE) if set(e) == {a, b})


def _tris(tri, c):
    row = [int(x) for x in tri[c] if x >= 0]
    return [tuple(row[i:i + 3]) for i in range(0, len(row), 3)]


def _face_rule(c, f):
    neg = [(c >> i) & 1 for i in range(8)]
    cs = FACE[f]
    fe = [_edge_of(cs[j], cs[(j + 1) % 4]) for j in range(4)]
    cross = [j for j in range(4) if neg[cs[j]] != neg[cs[(j + 1) % 4]]]
    if len(cross) == 2:
        return {frozenset((fe[cross[0]], fe[cross[1]]))}
    if len(cross) == 4:
        return {frozenset((fe[(j + 3) % 4], fe[j])) for j in range(4) if neg[cs[j]]}
    return set()


def _boundary(tris):
    """directed edges of the triangles that are not cancelled by the reverse edge of another triangle"""
    es = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
    s = set(es)
    return [e for e in es if (e[1], e[0]) not in s]


def test_table_uses_exactly_the_crossing_edges():
    tri, ntri = T.mc_table()
    for c in range(256):
        neg = [(c >> i) & 1 for i in range(8)]
        crossing = {i for i, (a, b) in enumerate(EDGE) if neg[a] != neg[b]}
        used = {e for t in _tris(tri, c) for e in t}
        assert used == crossing, c
        assert len(_tris(tri, c)) == ntri[c] <= 5


def test_table_face_segments_follow_the_face_rule():
    tri, _ = T.mc_table()
    for c in range(256):
        segs = {frozenset(e) for e in _boundary(_tris(tri, c))}
        want = set().union(*[_face_rule(c, f) for f in range(6)])
        assert segs == want, c


def _ambiguous(c):
    neg = [(c >> i) & 1 for i in range(8)]
    return any(sum(neg[f[j]] != neg[f[(j + 1) % 4]] for j in range(4)) == 4 for f in FACE)


def test_table_complementary_configurations_have_reversed_winding():
    tri, _ = T.mc_table()
    checked = 0
    for c in range(256):
        if _ambiguous(c):   # the face rule separates the negative corners, so an ambiguous face joins other edges in the complement
            continue
        rot = lambda t: min(t[i:] + t[:i] for i in range(3))
        a = {rot(t) for t in _tris(tri, c)}
        b = {rot(t[::-1]) for t in _tris(tri, 255 - c)}
        assert a == b, c
        checked += 1
    assert checked > 100


def _sphere_mesh(tri, n=24, r=0.37):
    """marching cubes of sdf = |p| - r on an n^3 grid of [-0.5, 0.5]^3 with the table; vertices keyed by global grid edge"""
    h = 1.0 / n
    g = (np.arange(n + 1) * h - 0.5)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    sdf = np.sqrt(X * X + Y * Y + Z * Z) - r
    tris, pos = [], {}
    for i, j, k in itertools.product(range(n), repeat=3):
        corners = [(i + a, j + b, k + c) for a, b, c in CORNER]
        s = [sdf[p] for p in corners]
        cfg = sum(1 << q for q in range(8) if s[q] < 0)
        for t in _tris(tri, cfg):
            ids = []
            for e in t:
                a, b = EDGE[e]
                key = tuple(sorted((corners[a], corners[b])))
                if key not in pos:
                    pa, pb = np.array(key[0]) * h - 0.5, np.array(key[1]) * h - 0.5
                    sa, sb = sdf[key[0]], sdf[key[1]]
                    pos[key] = pa + (sa / (sa - sb)) * (pb - pa)
                ids.append(key)
            tris.append(tuple(ids))
    return tris, pos, h


def test_sphere_mesh_is_closed_and_on_the_sphere():
    tri, _ = T.mc_table()
    tris, pos, h = _sphere_mesh(tri)
    assert len(tris) > 1000
    directed = {}
    for t in tris:
        for i in range(3):
            e = (t[i], t[(i + 1) % 3])
            directed[e] = directed.get(e, 0) + 1
    for (a, b), cnt in directed.items():
        assert cnt == 1 and directed.get((b, a)) == 1       # every undirected edge: two triangles, opposite directions
    r = np.array([np.linalg.norm(p) for p in pos.values()])
    assert np.abs(r - 0.37).max() < h
    # right-hand normals point inside (sdf < 0), so the PLY's reversed faces point outside
    for t in tris[:500]:
        a, b, c = (pos[k] for k in t)
        assert np.dot(np.cross(b - a, c - a), a + b + c) < 0


# ---- CPU: C-ABI boundary ---------------------------------------------------------------------------------------------------------
def test_capi_null_handles_are_refused(api):
    L = api.lib()
    null = C.c_void_p(None)
    d = C.c_double(0)
    u3 = (C.c_uint32 * 3)()
    i3 = (C.c_int32 * 3)(1, 1, 1)
    n = C.c_size_t(0)
    calls = [
        (L.lama_tsdm_create, (C.c_double(0.05), C.c_uint32(32), C.c_int(0), null, null, null, null)),
        (L.lama_tsdm_set_max_distance, (null, C.c_double(0.2))),
        (L.lama_tsdm_max_distance, (null, C.byref(d))),
        (L.lama_tsdm_insert_point_clouds, (null, null, null, C.c_int(0), null, null, null)),
        (L.lama_tsdm_distance, (null, null, C.c_int(0), null, null)),
        (L.lama_tsdm_bounds, (null, u3, u3, null)),
        (L.lama_tsdm_export, (null, u3, i3, null, null, null)),
        (L.lama_tsdm_to_mesh, (null, null, C.c_size_t(0), C.byref(n))),
        (L.lama_tsdm_write_ply, (null, C.c_char_p(b"x.ply"))),
        (L.lama_tsdm_kernel_times, (null, null, null)),
    ]
    for fn, args in calls:
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0
    assert L.lama_tsdm_destroy(null) == 0
    h = C.c_void_p()
    assert L.lama_tsdm_create(C.c_double(0.05), C.c_uint32(16), C.c_int(0), null, null, null, C.byref(h)) == -1   # patch_size != 32


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _room_clouds(synth, n, n_beams=1080, name="room", tilt=0.0):
    ds = synth.make_dataset(name, n, n_beams=n_beams)
    origins = np.c_[ds.truth[:, :2], np.zeros(n)]
    if tilt:
        quats = np.array([synth.quat_xyzw(t[2], tilt, 0.5 * tilt) for t in ds.truth])
    else:
        quats = np.array([_qz(t[2]) for t in ds.truth])
    return list(ds.scans), origins, quats


def _check_equal(g, o, is3d):
    ng, mng, mxg = g.bounds()
    no, mno, mxo = o.bounds()
    assert ng == no and np.array_equal(mng, mno) and np.array_equal(mxg, mxo)
    _, lo, size = _box(o, is3d)
    return _same_cells(g, o, lo, size)


@pytest.mark.gpu
def test_gpu_2d_room_per_cloud_and_batched_equal_oracle(gpu_api, synth):
    clouds, origins, quats = _room_clouds(synth, 300)
    o = T.Oracle(0.05)
    ro = o.insertPointClouds(clouds, origins, quats)
    g1 = gpu_api.TruncatedSignedDistanceMap(0.05)
    r1 = [g1.insertPointCloud(c, origins[k], quats[k]) for k, c in enumerate(clouds)]
    g2 = gpu_api.TruncatedSignedDistanceMap(0.05)
    r2 = g2.insertPointClouds(clouds, origins, quats)
    assert np.array_equal(ro, r1) and np.array_equal(ro, r2)
    ex = _check_equal(g1, o, False)
    _check_equal(g2, o, False)
    assert ex["on"].sum() > 10000


@pytest.mark.gpu
def test_gpu_2d_config4_all_scans_span_several_chunks(gpu_api, synth):
    clouds, origins, quats = _room_clouds(synth, 5000, name="loop")
    o = T.Oracle(0.05)
    ro = o.insertPointClouds(clouds, origins, quats)
    g = gpu_api.TruncatedSignedDistanceMap(0.05)
    assert np.array_equal(g.insertPointClouds(clouds, origins, quats), ro)
    _check_equal(g, o, False)
    _, launches = g.kernelTimes()
    assert launches["insert"] > 12      # more than one dedupe pass and more than one sort chunk


@pytest.mark.gpu
def test_gpu_2d_tilted_sensor_and_degenerate_mesh(gpu_api, synth):
    clouds, origins, quats = _room_clouds(synth, 60, tilt=0.03)
    o = T.Oracle(0.05)
    g = gpu_api.TruncatedSignedDistanceMap(0.05)
    assert np.array_equal(g.insertPointClouds(clouds, origins, quats), o.insertPointClouds(clouds, origins, quats))
    _check_equal(g, o, False)
    vg, idx = g.toMesh()
    vo = o.toMesh()
    assert len(vo) > 0 and np.array_equal(vg.view(np.uint32), vo.view(np.uint32)) and np.array_equal(idx, np.arange(len(vo)))
    assert np.abs(vg[:, 2] - F(-O * 0.05)).max() < 0.1     # the reference's 2-D mesh sits at z = (0 - offset) * resolution


@pytest.mark.gpu
@pytest.mark.parametrize("is3d", [False, True])
def test_gpu_distance_queries_equal_oracle(gpu_api, synth, is3d):
    rng = np.random.default_rng(21)
    if is3d:
        clouds, origins, quats = synth.make_clouds_3d(6, n_az=450)
        q = rng.uniform([-5, -5, 0], [5, 5, 3], (10000, 3))
    else:
        clouds, origins, quats = _room_clouds(synth, 40)
        q = np.c_[rng.uniform(-10, 10, (10000, 2)), np.zeros(10000)]
    o = T.Oracle(0.05, is3d)
    g = gpu_api.TruncatedSignedDistanceMap(0.05, is3d=is3d, center=(0, 0, 1.5))
    o.insertPointClouds(clouds, origins, quats)
    g.insertPointClouds(clouds, origins, quats)
    d1, g1 = g.distance(q, gradient=True)
    d2, g2 = o.distance(q, gradient=True)
    assert np.array_equal(d1, d2) and np.array_equal(g1, g2)
    assert (d1 != F(0.15)).sum() > 100


@pytest.mark.gpu
@pytest.mark.parametrize("res", [0.05, 0.1])
def test_gpu_3d_room_cells_mesh_and_ply_equal_oracle(gpu_api, synth, res, tmp_path):
    from iris_lama_b200 import sdm
    clouds, origins, quats = synth.make_clouds_3d(30)
    o = T.Oracle(res, True)
    g = gpu_api.TruncatedSignedDistanceMap(res, is3d=True, center=(0, 0, 1.5))
    assert np.array_equal(g.insertPointClouds(clouds, origins, quats), o.insertPointClouds(clouds, origins, quats))
    _check_equal(g, o, True)
    vg, _ = g.toMesh()
    vo = o.toMesh()
    assert len(vo) > 10000 and np.array_equal(vg.view(np.uint32), vo.view(np.uint32))
    assert sdm.export_to_ply(g, tmp_path / "g.ply") and o.write_ply(tmp_path / "o.ply")
    assert (tmp_path / "g.ply").read_bytes() == (tmp_path / "o.ply").read_bytes()


@pytest.mark.gpu
def test_gpu_weight_clamp_through_a_batch(gpu_api):
    cloud = np.array([[0.1, 0.0, 0.0], [0.0, 0.1, 0.0]])
    o = T.Oracle(0.05)
    g = gpu_api.TruncatedSignedDistanceMap(0.05)
    batch = [cloud] * 150
    assert np.array_equal(g.insertPointClouds(batch), o.insertPointClouds(batch))
    ex = _check_equal(g, o, False)
    assert ex["weight"].max() == F(10000)


@pytest.mark.gpu
def test_gpu_window_overflow_leaves_the_map_unchanged(gpu_api, synth):
    clouds, origins, quats = _room_clouds(synth, 10)
    g = gpu_api.TruncatedSignedDistanceMap(0.05, window=(8, 8, 1))      # 12.8 m: the 20 m room does not fit
    g.insertPointClouds([c[np.linalg.norm(c, axis=1) < 2.0] for c in clouds[:2]], origins[:2], quats[:2])
    n0, lo, size = _box(g, False)
    before = g.export(lo, size)
    with pytest.raises(gpu_api.LamaError) as e:
        g.insertPointClouds(clouds, origins, quats)
    assert e.value.code == -4
    n1, _, _ = g.bounds()
    after = g.export(lo, size)
    assert n1 == n0 and all(np.array_equal(before[k], after[k]) for k in before)


@pytest.mark.gpu
def test_gpu_same_batch_twice_is_byte_identical(gpu_api, synth):
    clouds, origins, quats = synth.make_clouds_3d(8, n_az=600)
    out = []
    for _ in range(2):
        g = gpu_api.TruncatedSignedDistanceMap(0.05, is3d=True, center=(0, 0, 1.5))
        g.insertPointClouds(clouds, origins, quats)
        _, lo, size = _box(g, True)
        out.append((g.export(lo, size), g.toMesh()[0]))
    for k in out[0][0]:
        assert np.array_equal(out[0][0][k].view(np.uint8), out[1][0][k].view(np.uint8))
    assert np.array_equal(out[0][1].view(np.uint32), out[1][1].view(np.uint32))
