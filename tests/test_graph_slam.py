"""GraphSlam2D (include/lama/graph_slam2d.h:51-173, src/graph_slam2d.cpp:104-430) and the Huber-robust pose-graph optimiser it runs.
CPU: the Huber loss of the PGO oracle (oracle/pose_graph_oracle.py) against closed forms and finite differences, the GraphSlam2D oracle
(oracle/graph_slam_oracle.py) against the rules of the reference's update, and the C-ABI boundary of the new entry points.  GPU: the device
optimiser (csrc/pgo.cu) and the device GraphSlam2D (csrc/frontend.cpp) against those oracles."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import pgo_oracle as pg
from oracle import pose_graph_oracle as pgg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PRIOR = pgg.diagonal([0.01, 0.01, 0.01])    # graph_slam2d.cpp:214
CHAIN = pgg.diagonal([0.25, 0.25, 0.15])    # :224
LOOP = pgg.huber(0.1)                       # :266


def _graph(n, loops, seed, outliers=0, loop_loss=LOOP):
    """a pose graph with GraphSlam2D's losses from synth.make_pose_graph; `outliers` loop edges get a gross error (2 m, 0.5 rad)"""
    from iris_lama_b200 import synth
    truth, nodes, edges = synth.make_pose_graph(n, loops, seed=seed, step=max(0.1, 100.0 / n))   # at least two and a half 40 m laps
    X = pg.from_xyr(nodes)
    chain = pg.to_xyr(pg.mul(pg.inv(X[:-1]), X[1:]))
    betweens = [(i, i + 1, chain[i], CHAIN) for i in range(n - 1)]
    rng = np.random.default_rng(seed + 100)
    for k, (a, b, m) in enumerate(edges):
        if k < outliers:
            m = m + np.array([2.0, -2.0, 0.5]) * rng.choice([-1.0, 1.0], 3)
        betweens.append((a, b, m, loop_loss))
    return truth, nodes, [(0, nodes[0], PRIOR)], betweens


# ---- Huber loss in the PGO oracle -------------------------------------------------------------------------------------------------------
def test_huber_weight_closed_form_on_both_sides_of_k():
    e = np.array([[0.03, -0.04, 0.0], [0.3, 0.0, -0.4], [0.0, 0.0, 0.0999]])   # |e| = 0.05, 0.5, 0.0999
    w0 = np.tile([4.0, 4.0, 10.0], (3, 1))
    w = pgg.loss_weights(e, w0, np.full(3, 0.1))
    assert np.allclose(w[0], 1.0) and np.allclose(w[2], 1.0)                 # |e| < k: weight 1
    assert np.allclose(w[1], math.sqrt(0.1 / 0.5))                            # |e| >= k: sqrt(k / |e|) on every row
    assert (pgg.loss_weights(e, w0, np.zeros(3)) == w0).all()                 # k = 0: the DiagonalLoss rows 1 / sigma


def test_huber_normal_equations_are_the_gradient_of_the_weighted_error():
    """with the Huber weights frozen at the linearisation point, b = -J^T r is minus the gradient of 1/2 sum w |e|^2 (to the O(|e|) of
    miniSAM's Jacobians, which leave out the derivative of the logarithm): errors ~1e-3 against k = 1e-4 keep both branches active"""
    rng = np.random.default_rng(4)
    n = 12
    truth = np.cumsum(rng.uniform(-0.5, 0.5, (n, 3)), 0)
    Xt = pg.from_xyr(truth)
    bt = []
    for a, b in [(i, i + 1) for i in range(n - 1)] + [(0, 6), (2, 9), (3, 11), (1, 7)]:
        m = pg.to_xyr(pg.mul(pg.inv(Xt[a:a + 1]), Xt[b:b + 1]))[0]
        bt.append((a, b, m, pgg.huber(1e-4) if b != a + 1 else CHAIN))
    bt[-1] = (1, 7, bt[-1][2], pgg.huber(1.0))                                # one factor below its k
    g = pgg.PoseGraph(truth + rng.normal(0, 1e-3, (n, 3)), [(0, truth[0], PRIOR)], bt)
    X = g.nodes
    _, rb, _, wb = g._errors(X, g.pri, g.btw)
    hub = g.btw[4] > 0
    nrm = np.linalg.norm(rb / wb, axis=1)
    assert (nrm[hub] > g.btw[4][hub]).any() and (nrm[hub] < g.btw[4][hub]).any()   # both Huber branches
    A, b = g._linearize(X, g.pri, g.btw)

    def f(Xp):   # 1/2 sum w |e|^2 with w frozen
        ep = pg.log(pg.mul(pg.inv(g.pri[1]), Xp[g.pri[0]])) * g.pri[2]
        eb = pg.log(pg.mul(pg.inv(g.btw[2]), pg.mul(pg.inv(Xp[g.btw[0]]), Xp[g.btw[1]]))) * wb
        return 0.5 * ((ep * ep).sum() + (eb * eb).sum())
    h = 1e-7
    grad = np.zeros(3 * n)
    for i in range(3 * n):
        d = np.zeros((n, 3)); d[i // 3, i % 3] = h
        grad[i] = (f(pg.mul(X, pg.exp(d))) - f(pg.mul(X, pg.exp(-d)))) / (2 * h)
    assert np.abs(b + grad).max() < 2e-2 * np.abs(grad).max()


def test_huber_below_k_is_the_unit_diagonal_loss():
    _, nodes, pri, bt = _graph(200, 100, seed=5, loop_loss=pgg.huber(1e3))
    g1 = pgg.PoseGraph(nodes, pri, bt)
    g2 = pgg.PoseGraph(nodes, pri, [(a, b, m, pgg.diagonal([1.0, 1.0, 1.0]) if l[1] > 0 else l) for a, b, m, l in bt])
    assert g1.optimize() and g2.optimize()
    assert g1.iterations == g2.iterations and g1.accepted == g2.accepted and (g1.nodes == g2.nodes).all()


def test_huber_resists_a_gross_outlier_loop_edge():
    unit = pgg.diagonal([1.0, 1.0, 1.0])
    moved = {}
    for name, loss in (("huber", LOOP), ("gauss", unit)):
        sol = []
        for outliers in (0, 1):
            _, nodes, pri, bt = _graph(400, 300, seed=5, outliers=outliers, loop_loss=loss)
            g = pgg.PoseGraph(nodes, pri, bt)
            assert g.optimize() and g.status == 0
            sol.append(g.nodes_xyr())
        moved[name] = np.abs(sol[1] - sol[0])[:, :2].max()
    assert moved["huber"] < 0.2 * moved["gauss"], moved


@pytest.mark.parametrize("n,loops,fixed", [(400, 300, False), (400, 300, True), (1200, 1500, False)])
def test_simple_pgo_graph_through_the_general_oracle_is_simple_pgo(n, loops, fixed):
    """SimplePGO's graph (simple_pgo.cpp:50-83) given to PoseGraph as an explicit factor list reproduces pgo_oracle.SimplePGO bit for bit:
    the general optimiser adds the losses and nothing else"""
    from iris_lama_b200 import synth
    truth, nodes, edges = synth.make_pose_graph(n, loops, seed=5)
    fl = [(0, truth[0]), (n // 2, truth[n // 2])] if fixed else []
    X = pg.from_xyr(nodes)
    priors = [(i, p, pgg.diagonal([0.1, 0.1, 0.1])) for i, p in fl] if fixed else [(0, X[0], pgg.diagonal([1.0, 1.0, 1.0]))]
    odom = pgg.diagonal([0.5, 0.5, 0.1])
    chain = pg.mul(pg.inv(X[:-1]), X[1:])
    betweens = [(i, i + 1, chain[i], odom) for i in range(n - 1)] + [(a, b, m, odom) for a, b, m in edges]
    s, g = pg.SimplePGO(nodes, edges, fl), pgg.PoseGraph(nodes, priors, betweens)
    assert s.optimize() and g.optimize()
    assert (g.iterations, g.lambda_tries, g.errors) == (s.iterations, s.lambda_tries, s.errors) and (g.nodes == s.nodes).all()


# ---- the GraphSlam2D oracle --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def two_laps(po, synth):
    from oracle import graph_slam_oracle as gso
    ds = synth.make_dataset("loop", 1600, n_beams=360)
    g = gso.GraphSlam2D()
    g.Init(*ds.truth[0])
    for t in range(ds.n_scans):
        g.update(ds.scans[t], ds.odom[t], float(t))
    return g


def test_oracle_key_poses_are_spaced_by_the_key_pose_rule(two_laps):
    g = two_laps
    _, orig = g.key_poses()
    X = pg.from_xyr(orig)
    d = pg.mul(pg.inv(X[1:]), X[:-1])
    far = np.hypot(d[:, 2], d[:, 3]) >= g.opt["key_pose_distance"]
    turned = np.abs(np.arctan2(d[:, 1], d[:, 0])) >= g.opt["key_pose_angular_distance"]
    assert len(orig) > 100 and (far | turned).all()


def test_oracle_loop_search_rules(two_laps):
    g = two_laps
    first = max(g.opt["key_pose_head_delay"], g.opt["ignore_n_chain_poses"])
    for r in g.decisions:
        if r["searched"]:
            assert r["key"] is not None and r["key"] >= first                # no search before key max(head_delay, ignore_n)
        else:
            assert not r["correlations"] and r["link"] is None
        if r["link"] is not None:                                             # at most one factor per update: the search stops at it
            assert r["correlations"][-1]["candidate"] == r["link"][0] and r["link"][1] == r["key"] - g.opt["key_pose_head_delay"]
        for i, c in enumerate(r["correlations"]):                             # the coarse retry is for the closest candidate only
            assert c["coarse_rmse"] is None or (i == 0 and c["rmse"] > g.opt["loop_closure_scan_rmse"])
    assert len(g.links) == sum(r["link"] is not None for r in g.decisions)


def test_oracle_optimises_exactly_when_the_flush_rule_says(two_laps):
    g = two_laps
    for r in g.decisions:
        if r["searched"]:
            want = r["queue"] > 0 and not (r["queue"] <= 5 and r["factordist"] <= 15.0)
            assert r["flush"] == want and (r["pgo"] is not None) == want
        else:
            assert not r["flush"]
    assert len(g.optimizations) == sum(r["flush"] for r in g.decisions)


def test_oracle_closes_loops_on_the_second_lap(two_laps):
    g = two_laps
    n = len(g.keys)
    assert any(ref > n // 2 for _, ref in g.links)
    assert sum(o[0] == 0 for o in g.optimizations) >= 1
    assert min(m for _, m in g.margins) > 1e-5


# ---- C-ABI ---------------------------------------------------------------------------------------------------------------------------------
def test_graph_options_struct_matches_the_header(api, tmp_path):
    src = tmp_path / "sz.cpp"
    src.write_text('#include "lama_b200.h"\n#include <cstddef>\n#include <cstdio>\nint main(){printf("%zu %zu %zu\\n", sizeof(lama_graph_options), '
                   'offsetof(lama_graph_options, loop_closure_scan_rmse), offsetof(lama_graph_options, ignore_n_chain_poses));}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["g++", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(api.GraphOptions), api.GraphOptions.loop_closure_scan_rmse.offset, api.GraphOptions.ignore_n_chain_poses.offset]


def test_graph_defaults_are_the_reference_defaults(api):
    o = api.GraphSlam2D.Options()
    # graph_slam2d.h:62-86
    assert (o.key_pose_distance, o.key_pose_angular_distance, o.key_pose_head_delay) == (1.0, 0.5 * math.pi, 5)
    assert (o.loop_search_max_distance, o.loop_search_min_distance, o.loop_max_candidates) == (10.0, 2.0, 5)
    assert (o.loop_closure_scan_rmse, o.loop_closure_max_candidates, o.ignore_n_chain_poses) == (0.05, 10, 20)
    s = o.slam   # Options : Slam2D::Options (slam2d.h:91-125)
    assert (s.trans_thresh, s.rot_thresh, s.l2_max, s.resolution, s.patch_size, s.max_iter, s.truncated_ray, s.transient_map) == (0.5, 0.5, 0.5, 0.05, 32, 100, 0.0, 0)
    assert api.GraphSlam2D.Options(l2_max=1.0, key_pose_head_delay=3, device=0).slam.l2_max == 1.0


def test_new_entry_points_refuse_null_arguments(api):
    L = api.lib()
    null = C.c_void_p(None)
    n = C.c_int(0)
    xyr = (C.c_double * 3)()
    pts = (C.c_double * 3)()
    calls = [
        (L.lama_graph_options_default, (null,)),
        (L.lama_graph_create, (null, null)),
        (L.lama_graph_set_pose, (null, xyr)),
        (L.lama_graph_update, (null, pts, C.c_int(1), null, null, xyr, C.c_double(0), null)),
        (L.lama_graph_get_pose, (null, xyr)),
        (L.lama_graph_get_key_poses, (null, null, null, null, C.c_int(0), C.byref(n))),
        (L.lama_graph_get_key_cloud, (null, C.c_int(0), null, C.c_int(0), null, null, C.byref(n))),
        (L.lama_graph_get_links, (null, null, C.c_int(0), C.byref(n))),
        (L.lama_graph_get_last_candidates, (null, null, C.c_int(0), C.byref(n))),
        (L.lama_graph_get_stats, (null, null, null, null)),
        (L.lama_graph_slam, (null, null)),
        (L.lama_pgo_optimize_graph, (C.c_int(0), null, C.c_int(3), null, null, null, C.c_int(0), null, null, null, C.c_int(0), null, null, null, C.c_int(0), null)),
    ]
    for fn, args in calls:
        fn.restype = C.c_int
        assert fn(*args) == -1, fn.__name__
        assert len(L.lama_last_error()) > 0
    o = api.GraphOptions()
    assert L.lama_graph_create(C.byref(o), null) == -1
    assert L.lama_graph_destroy(null) == 0


def test_pgo_optimize_graph_validates_before_touching_a_device(api):
    with pytest.raises(api.LamaError) as e:      # out-of-range node
        api.pgo_optimize_graph(np.zeros((3, 3)), [(0, [0, 0, 0], api.diagonal_loss([1, 1, 1]))], [(0, 5, [1, 0, 0], api.huber_loss(0.1))])
    assert e.value.code == -1
    with pytest.raises(api.LamaError) as e:      # a diagonal loss with a zero sigma
        api.pgo_optimize_graph(np.zeros((3, 3)), [(0, [0, 0, 0], api.diagonal_loss([1, 0, 1]))], [])
    assert e.value.code == -1


def test_graph_needs_a_gpu_or_fails_loudly(api):
    if api.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(api.LamaError) as e:
        api.GraphSlam2D()
    assert e.value.code == -3                    # LAMA_ERR_NO_DEVICE
    with pytest.raises(api.LamaError) as e:
        api.pgo_optimize_graph(np.zeros((3, 3)), [(0, [0, 0, 0], api.diagonal_loss([1, 1, 1]))], [(0, 1, [1, 0, 0], api.huber_loss(0.1))])
    assert e.value.code == -3


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------------
def _api_factors(api, pri, bt):
    conv = lambda l: api.huber_loss(l[1]) if l[1] > 0 else api.diagonal_loss(1.0 / l[0])
    return [(i, m, conv(l)) for i, m, l in pri], [(a, b, m, conv(l)) for a, b, m, l in bt]


@pytest.mark.gpu
@pytest.mark.parametrize("n,loops,outliers", [(200, 150, 2), (2000, 3000, 5)])
def test_device_pgo_graph_equals_oracle(gpu_api, n, loops, outliers):
    _, nodes, pri, bt = _graph(n, loops, seed=21, outliers=outliers)
    o = pgg.PoseGraph(nodes, pri, bt)

    def loop_errors(X):
        _, rb, _, wb = o._errors(X, o.pri, o.btw)
        return np.linalg.norm(rb / wb, axis=1)[o.btw[4] > 0]
    start = loop_errors(o.nodes)
    o_ok = o.optimize()
    end = loop_errors(o.nodes)
    assert (start > 0.1).any() and (end > 0.1).sum() >= outliers and (end < 0.1).any()   # both Huber branches are taken
    status, x, rep, acc = gpu_api.pgo_optimize_graph(nodes, *_api_factors(gpu_api, pri, bt))
    assert o_ok and status == o.status == 0
    assert rep["iterations"] == o.iterations and rep["lambda_tries"] == o.lambda_tries and acc == o.accepted
    assert abs(rep["initial_error"] - o.errors[0]) < 1e-9 * o.errors[0]
    d = x - o.nodes_xyr()
    d[:, 2] = (d[:, 2] + np.pi) % (2 * np.pi) - np.pi
    assert np.abs(d).max() < 1e-6


@pytest.mark.gpu
def test_device_pgo_graph_10k_nodes_is_repeatable_and_reduces_the_error(gpu_api):
    truth, nodes, pri, bt = _graph(10000, 40001, seed=11, outliers=20)
    p, b = _api_factors(gpu_api, pri, bt)
    s1, x1, r1, a1 = gpu_api.pgo_optimize_graph(nodes, p, b)
    s2, x2, r2, a2 = gpu_api.pgo_optimize_graph(nodes, p, b)
    assert s1 == 0 and r1["final_error"] < 1e-2 * r1["initial_error"]
    assert (s2, r2["iterations"], r2["cg_iterations"], a2) == (s1, r1["iterations"], r1["cg_iterations"], a1) and (x1 == x2).all()
    assert np.abs(x1 - truth)[:, :2].max() < np.abs(nodes - truth)[:, :2].max()


@pytest.mark.gpu
def test_device_graph_slam_two_laps_equals_oracle(gpu_api, po, synth):
    from oracle import graph_slam_oracle as gso
    ds = synth.make_dataset("loop", 1600, n_beams=1080)
    o = gso.GraphSlam2D()
    g = gpu_api.GraphSlam2D()
    o.Init(*ds.truth[0]); g.Init(*ds.truth[0])
    slam = g.slam
    n_links = n_opts = 0
    for t in range(ds.n_scans):
        n_dec = len(o.decisions)
        uo, ug = o.update(ds.scans[t], ds.odom[t], float(t)), g.update(ds.scans[t], ds.odom[t], float(t))
        assert uo == ug, t
        if not uo:
            continue
        so, sg = o.slam.state(), slam.getPose()
        assert abs(so[2] - sg[0]) < 1e-9 and abs(so[3] - sg[1]) < 1e-9 and abs(math.atan2(so[1], so[0]) - sg[2]) < 1e-9, t
        rec = o.decisions[n_dec]
        st = g.stats()
        assert st["key_poses"] == len(o.keys), t
        assert g.lastCandidates().tolist() == rec["candidates"], t
        assert [tuple(l) for l in g.links().tolist()] == o.links, t
        assert st["loop_factors"] == len(o.links)
        assert st["optimizations"] == len(o.optimizations) and st["optimizations_ok"] == sum(p[0] == 0 for p in o.optimizations), t
        if rec["pgo"] is not None:
            assert st["last_status"] == rec["pgo"][0] and st["last_report"]["iterations"] == rec["pgo"][1], t
            assert st["last_report"]["lambda_tries"] == rec["pgo"][2], t
        assert np.abs(g.getPose() - o.getPose()).max() < 1e-6, t
    cor_g, org_g, stamps = g.keyPoses()
    cor_o, org_o = o.key_poses()
    assert np.abs(org_g - org_o).max() < 1e-9 and np.abs(cor_g - cor_o).max() < 1e-6
    assert stamps.tolist() == [k["stamp"] for k in o.keys]
    assert min(m for _, m in o.margins) > 1e-5          # a flipped decision would point at an ill-conditioned scenario
    st = g.stats()
    assert st["loop_factors"] >= 5 and st["optimizations_ok"] >= 1
    assert np.abs(cor_g - org_g).max() > 1e-4           # the correction is not the identity
    pts, org, q = g.keyCloud(3)
    assert (pts == ds.scans[[int(s) for s in stamps][3]]).all() and (q == [0, 0, 0, 1]).all()
    assert gpu_api.lib().lama_slam_destroy(slam.h) == 0 and slam.getPose().shape == (3,)   # destroying the borrowed handle is a no-op
