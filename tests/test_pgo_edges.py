"""The pose-graph optimiser (csrc/pgo.cu: k_pgo_linearize, k_pgo_assemble, the cooperative k_pgo_pcg, k_pgo_retract, k_pgo_error_*, and the
host LM loop of pgo_optimize_graph) at its edges.

CPU: the SE2 maps of the oracle (oracle/pgo_oracle.py) and of the host build of lama_core.h (tests/emu) against 50-digit mpmath; the LM
schedule when a damped diagonal block is zero; the refusal of self-loop factors; and a numpy restatement of k_pgo_pcg
(pose_graph_oracle.pcg) on long chains with few loops, whose iteration counts must stay 10 % below the cap of 4 n + 200.
GPU: the device against the oracle (oracle/pose_graph_oracle.py) on unreferenced nodes, duplicate and reversed loop edges, headings at +-pi,
far-off coordinates, tiny graphs, Huber edges, long chains and a lowered PCG cap.  Every device case runs twice and must return the same bits."""
import ctypes as C
import math
import os
import subprocess

import mpmath as mp
import numpy as np
import pytest

from oracle import pgo_oracle as pg
from oracle import pose_graph_oracle as pgg

HERE = os.path.dirname(os.path.abspath(__file__))
EPS = 2.0 ** -52
PI = math.pi

SIMPLE = dict(prior=pgg.diagonal([1.0, 1.0, 1.0]), chain=pgg.diagonal([0.5, 0.5, 0.1]), loop=pgg.diagonal([0.5, 0.5, 0.1]))   # simple_pgo.cpp:52-82
GRAPH = dict(prior=pgg.diagonal([0.01, 0.01, 0.01]), chain=pgg.diagonal([0.25, 0.25, 0.15]), loop=pgg.huber(0.1))              # graph_slam2d.cpp:214-266


# ---- fixtures ------------------------------------------------------------------------------------------------------------------------------
def lap_graph(n=400, loops=300, seed=3, offset=(0.0, 0.0), w=SIMPLE):
    """synth.make_pose_graph's laps as an explicit factor list (prior on node 0, odometry chain, loop edges), translated by `offset`"""
    from iris_lama_b200 import synth
    _, nodes, edges = synth.make_pose_graph(n, loops, seed=seed)
    nodes = nodes + [offset[0], offset[1], 0.0]
    X = pg.from_xyr(nodes)
    chain = pg.to_xyr(pg.mul(pg.inv(X[:-1]), X[1:]))
    bt = [(i, i + 1, chain[i], w["chain"]) for i in range(n - 1)] + [(a, b, m, w["loop"]) for a, b, m in edges]
    return nodes, [(0, nodes[0], w["prior"])], bt


def long_chain(n, loops, w, seed=0):
    """one circular lap of n nodes 0.1 m apart, odometry with noise, loop edges (0, n-1) and (n/3, 2n/3) from the truth; without loops
    the prior is moved off node 0 so that the whole chain has to follow it"""
    rng = np.random.default_rng(seed)
    ang = 2 * np.pi * np.arange(n) / n
    R = n * 0.1 / (2 * np.pi)
    truth = np.stack([R * np.cos(ang), R * np.sin(ang), ang + np.pi / 2], 1)
    Xt = pg.from_xyr(truth)
    rel = pg.to_xyr(pg.mul(pg.inv(Xt[:-1]), Xt[1:])) + rng.normal(0, [0.02, 0.02, 0.004], (n - 1, 3))
    Rel = pg.from_xyr(rel)
    X = np.zeros((n, 4))
    X[0] = Xt[0]
    for i in range(n - 1):
        X[i + 1] = pg.mul(X[i:i + 1], Rel[i:i + 1])[0]
    nodes = pg.to_xyr(X)
    bt = [(i, i + 1, rel[i], w["chain"]) for i in range(n - 1)]
    for a, b in [(0, n - 1), (n // 3, 2 * n // 3)][:loops]:
        bt.append((a, b, pg.to_xyr(pg.mul(pg.inv(Xt[a:a + 1]), Xt[b:b + 1]))[0] + rng.normal(0, [0.01, 0.01, 0.002]), w["loop"]))
    prior = truth[0] + ([0.3, -0.2, 0.05] if loops == 0 else 0.0)
    return nodes, [(0, prior, w["prior"])], bt


def with_unreferenced_node(nodes, pri, bt, at):
    """insert a node that no factor references at index `at`"""
    sh = lambda i: i + (i >= at)
    nodes = np.insert(nodes, at, [[1.5, -2.5, 0.7]], axis=0)
    return nodes, [(sh(i), m, l) for i, m, l in pri], [(sh(a), sh(b), m, l) for a, b, m, l in bt]


def wrap(d):
    d = np.array(d, float)
    d[..., 2] = (d[..., 2] + np.pi) % (2 * np.pi) - np.pi
    return d


@pytest.fixture(scope="module")
def emu():
    subprocess.check_call(["make", "-C", os.path.join(HERE, "emu"), "-s"])
    L = C.CDLL(os.path.join(HERE, "emu", "_build", "liblama_emu.so"))
    L.emu_se2.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]

    def call(op, a, b=None):
        a = np.ascontiguousarray(a, float)
        b = None if b is None else np.ascontiguousarray(b, float)
        out = np.zeros(4)
        L.emu_se2(op, a.ctypes.data, None if b is None else b.ctypes.data, out.ctypes.data)
        return out
    return call


# ---- SE2 against 50-digit mpmath -----------------------------------------------------------------------------------------------------------
mp.mp.dps = 50
_NA = np.nextafter
THETAS = [0.0, 1e-12, -1e-12, _NA(1e-10, 0), 1e-10, -1e-10, _NA(1e-10, 1), 1e-8, 1e-5, math.sqrt(2e-10), 1e-4, 1e-3, 0.1, 1.0, -2.5, 3.0,
          _NA(PI, 0), PI, -PI, _NA(-PI, 0)]
TRANS = [(0.3, -0.7), (1e5, -3e4), (-2.0, 1e5)]


def _mp_exp(v):
    th = mp.mpf(v[2])
    c, s = mp.cos(th), mp.sin(th)
    a, b = (mp.mpf(1), mp.mpf(0)) if th == 0 else (s / th, (1 - c) / th)
    return [c, s, a * v[0] - b * v[1], b * v[0] + a * v[1]], a, b


def _mp_log(X):
    c, s = mp.mpf(X[0]), mp.mpf(X[1])
    r = mp.sqrt(c * c + s * s)
    c, s = c / r, s / r
    th = mp.atan2(s, c)
    h = mp.mpf(1) if th == 0 else (th / 2) * s / (1 - c)
    return [h * X[2] + th / 2 * X[3], -th / 2 * X[2] + h * X[3], th], h


def _exp_formula(v, c, s):
    """se2.hpp:389-412 outside the series branch, in fp64 from the fp64 (c, s)"""
    a, b = s / v[2], (1.0 - c) / v[2]
    return a * v[0] - b * v[1], b * v[0] + a * v[1]


def _log_formula(X):
    """se2.hpp:519-542 outside the series branch, in fp64"""
    th = math.atan2(X[1], X[0])
    half = 0.5 * th
    h = -(half * X[1]) / (X[0] - 1.0)
    return h * X[2] + half * X[3], -half * X[2] + h * X[3]


def test_se2_exp_against_mpmath(emu):
    """exp: c, s within 3 ulps of cos, sin; t within 4 ulps of |a v0| + |b v1|, except where (1 - c) / theta cancels (1e-10 <= |theta| below
    about 0.1, outside the series branch): there the result must be the reference formula in fp64, and its distance from the true value is
    bounded by the rounding of c, 2.5 eps / |theta| |v1|.  Measured there: 5.0e-4 m at |v| = 1e5 m and theta = 1e-8, where 1 - c rounds
    to 0 or 1 ulp instead of 5e-17."""
    worst = 0.0
    for th in THETAS:
        for v0, v1 in TRANS:
            v = np.array([v0, v1, th])
            want, a, b = _mp_exp(v)
            for name, got in (("oracle", pg.exp(v)[0]), ("emu", emu(2, v))):
                for k in (0, 1):
                    assert abs(got[k] - want[k]) <= 3 * EPS * abs(want[k]), (name, th, k)
                scale = {2: float(abs(a * v0) + abs(b * v1)), 3: float(abs(b * v0) + abs(a * v1))}
                db = 0.0 if abs(th) < 1e-10 else 2.5 * EPS / abs(th)        # error of b = (1 - c) / theta from the rounding of c
                cancel = {2: db * abs(v1), 3: db * abs(v0)}
                for k in (2, 3):
                    err = float(abs(got[k] - want[k]))
                    assert err <= 4 * EPS * scale[k] + cancel[k], (name, th, v0, v1, k, err)
                if any(cancel[k] > 4 * EPS * scale[k] for k in (2, 3)):
                    assert tuple(got[2:]) == _exp_formula(v, got[0], got[1]), (name, th)
                    worst = max(worst, float(max(abs(got[2] - want[2]), abs(got[3] - want[3]))))
    assert 4e-4 < worst < 5.1e-4


def test_se2_log_against_mpmath(emu):
    """log of the oracle and of lama_core.h's se2_log (what k_pgo_linearize takes every factor error with) on (cos theta, sin theta, t) built
    by from_xyr: theta within 2 ulps; upsilon within 4 ulps of |h t| + |theta / 2| |t| except where -(theta / 2 s) / (c - 1) cancels: c - 1 is
    exact, but the rounding of (c, s) to a unit vector, about eps, is divided by |c - 1|.  There the result must be the reference formula in
    fp64 and within 2.5 eps / |c - 1| |h| |t| of the true value.  Measured: below 2e-6 relative to |t|, the largest just above the series
    switch (|c - 1| = 1e-10).  c - 1 on both sides of -1e-10 picks the branch; the series term is 1 - theta^2 / 12 in the oracle and
    1 - (1 / 12) theta theta in lama_core.h, each checked against its own fp64 restatement and both against mpmath."""
    cs = [1.0 - 1e-10 + k * 2.0 ** -53 for k in range(-3, 4)]
    states = [pg.from_xyr([0, 0, th])[0] for th in THETAS if abs(abs(th) - PI) > 0] + [np.array([c, math.sqrt(1 - c * c), 0, 0]) for c in cs]
    worst = 0.0
    for X0 in states:
        for t0, t1 in TRANS:
            X = np.array([X0[0], X0[1], t0, t1])
            want, h = _mp_log(X)
            for name, got in (("oracle", pg.log(X[None])[0]), ("emu", emu(4, X))):
                assert abs(got[2] - want[2]) <= 2 * EPS * abs(want[2]), (name, X)
                series = abs(X[0] - 1.0) < 1e-10
                tn = abs(t0) + abs(t1)
                scale = float(abs(h) * tn + abs(want[2]) / 2 * tn)
                cancel = 0.0 if series else 2.5 * EPS / abs(X[0] - 1.0) * float(abs(h)) * tn
                for k in (0, 1):
                    err = float(abs(got[k] - want[k]))
                    assert err <= 4 * EPS * scale + cancel, (name, X, k, err)
                if cancel > 4 * EPS * scale:
                    assert tuple(got[:2]) == _log_formula(X), (name, X)
                    worst = max(worst, max(float(abs(got[k] - want[k])) for k in (0, 1)) / tn)
    assert worst < 2e-6
    # the series switch: |c - 1| < 1e-10 takes the series term, otherwise the formula
    for c in cs:
        X = np.array([c, math.sqrt(1 - c * c), 1.0, 0.0])
        th = math.atan2(X[1], X[0])
        formula = -(0.5 * th * X[1]) / (c - 1.0)
        series = abs(c - 1.0) < 1e-10
        assert pg.log(X[None])[0][0] == (1.0 - th * th / 12.0 if series else formula)
        assert emu(4, X)[0] == (1.0 - (1.0 / 12.0) * th * th if series else formula)
    assert any(abs(c - 1.0) < 1e-10 for c in cs) and any(abs(c - 1.0) >= 1e-10 for c in cs)


def test_se2_log_at_pi_takes_the_sign_of_s(emu):
    """c = -1, s = +-0: atan2 gives +-pi, h = 0, and upsilon = +-pi / 2 (t1, -t0): the sign of s (a signed zero) picks the branch, in the
    oracle and in lama_core.h"""
    for s, sign in ((0.0, 1.0), (-0.0, -1.0)):
        X = np.array([-1.0, s, 2.0, -3.0])
        for got in (pg.log(X[None])[0], emu(4, X)):
            assert got[2] == sign * PI
            assert got[0] == sign * PI / 2 * -3.0 and got[1] == -sign * PI / 2 * 2.0
    for th in (PI, -PI, _NA(PI, 0)):   # from_xyr(+-pi) is not c = -1, s = 0: s = +-1.2e-16 keeps the sign of theta
        X = pg.from_xyr([0, 0, th])
        assert X[0, 0] == -1.0 and math.copysign(1.0, X[0, 1]) == math.copysign(1.0, th)
        assert pg.log(X)[0, 2] == math.atan2(X[0, 1], X[0, 0]) == emu(4, np.append(X[0, :2], [0.0, 0.0]))[2]


def test_se2_mul_inv_adj_against_mpmath(emu):
    """mul and inv of the oracle and of lama_core.h within 4 ulps of the sum of the magnitudes of their terms, translations up to 1e5 m;
    Adj is a rearrangement of the state, checked exactly"""
    rng = np.random.default_rng(9)
    for th1 in THETAS:
        th2 = float(rng.uniform(-3, 3))
        for (a0, a1), (b0, b1) in zip(TRANS, TRANS[1:] + TRANS[:1]):
            A, B = pg.from_xyr([a0, a1, th1])[0], pg.from_xyr([b0, b1, th2])[0]
            mA, mB = [mp.mpf(x) for x in A], [mp.mpf(x) for x in B]
            want_mul = [mA[0] * mB[0] - mA[1] * mB[1], mA[0] * mB[1] + mA[1] * mB[0],
                        mA[2] + mA[0] * mB[2] - mA[1] * mB[3], mA[3] + mA[1] * mB[2] + mA[0] * mB[3]]
            r = mp.sqrt(want_mul[0] ** 2 + want_mul[1] ** 2)
            want_mul[0] /= r; want_mul[1] /= r
            sc = [1.0, 1.0, abs(A[2]) + abs(B[2]) + abs(B[3]), abs(A[3]) + abs(B[2]) + abs(B[3])]
            r = mp.sqrt(mA[0] ** 2 + mA[1] ** 2)
            ic, is_ = mA[0] / r, -mA[1] / r
            want_inv = [ic, is_, -(ic * mA[2] - is_ * mA[3]), -(is_ * mA[2] + ic * mA[3])]
            isc = [1.0, 1.0, abs(A[2]) + abs(A[3]), abs(A[2]) + abs(A[3])]
            for name, gm, gi in (("oracle", pg.mul(A[None], B[None])[0], pg.inv(A[None])[0]), ("emu", emu(0, A, B), emu(1, A))):
                for k in range(4):
                    assert float(abs(gm[k] - want_mul[k])) <= 4 * EPS * sc[k], (name, th1, k)
                    assert float(abs(gi[k] - want_inv[k])) <= 4 * EPS * isc[k], (name, th1, k)
            M = pg.adj(A[None])[0]
            assert (M == [[A[0], -A[1], A[3]], [A[1], A[0], -A[2]], [0, 0, 1]]).all()


# ---- the LM schedule and refusals ---------------------------------------------------------------------------------------------------------------
def test_oracle_zero_block_makes_ten_tries_and_leaves_the_nodes():
    """a node no factor references has a zero diagonal block; lambda * 0 = 0, so every try fails like the reference's zero pivot
    (RANK_DEFICIENCY): lambda = 1e-5 * 2^(k (k + 1) / 2) for k = 0..9, then 3.5e11 >= 1e10 ends the iteration in ERROR_INCREASE"""
    nodes, pri, bt = with_unreferenced_node(*lap_graph(), at=200)
    g = pgg.PoseGraph(nodes, pri, bt)
    assert not g.optimize()
    assert (g.status, g.iterations, g.lambda_tries, g.accepted) == (2, 1, 10, [0] * 10)
    assert g.lambdas == [1e-5 * 2.0 ** (k * (k + 1) // 2) for k in range(10)]
    assert (g.nodes == pg.from_xyr(nodes)).all()


def test_self_loops_are_refused_by_both_oracles_and_the_c_abi(api):
    nodes, pri, bt = lap_graph(60, 0)
    with pytest.raises(ValueError):
        pgg.PoseGraph(nodes, pri, bt + [(7, 7, [0.1, 0, 0], SIMPLE["loop"])])
    with pytest.raises(ValueError):
        pg.SimplePGO(nodes, [(3, 9, [0.1, 0, 0]), (9, 9, [0.1, 0, 0])])
    # the C ABI refuses them while validating its arguments, before any device call (the same error with or without a GPU)
    with pytest.raises(api.LamaError) as e:
        api.pgo_optimize_graph(nodes, [(0, nodes[0], api.diagonal_loss([1, 1, 1]))], [(0, 1, [0.1, 0, 0], api.diagonal_loss([1, 1, 1])),
                                                                                      (4, 4, [0.1, 0, 0], api.huber_loss(0.1))])
    assert e.value.code == -1 and "distinct" in str(e.value)
    with pytest.raises(api.LamaError) as e:
        api.SimplePGO(nodes, [(3, 9, [0.1, 0, 0]), (9, 9, [0.1, 0, 0])]).optimize()
    assert e.value.code == -1 and "distinct" in str(e.value)


def test_oracle_with_a_pcg_cap_of_one_rejects_every_try():
    nodes, pri, bt = lap_graph()
    g = pgg.PoseGraph(nodes, pri, bt, cg_cap=1)
    assert not g.optimize() and (g.status, g.iterations, g.lambda_tries, g.accepted) == (2, 1, 10, [0] * 10)
    assert g.cg_iterations == [1] * 10 and (g.nodes == pg.from_xyr(nodes)).all()


def pick_pcg_cap(nodes, pri, bt):
    """a cap a few iterations below what the first solve needs, at which every try's decision (truncated or not) is at least 3 iterations
    clear of the cap, so that the device's fixed-order sums cannot flip it"""
    free = pgg.PoseGraph(nodes, pri, bt, cg_cap=4 * len(nodes) + 200)
    free.optimize()
    first = free.cg_iterations[0]
    for cap in range(first - 3, first - 90, -3):
        systems = []
        o = pgg.PoseGraph(nodes, pri, bt, cg_cap=cap)
        o.optimize(on_solve=lambda A, b, lam: systems.append((A, b, lam)))
        need = [pgg.pcg(A, b, lam)[1] for A, b, lam in systems]
        if o.status == 0 and o.lambda_tries > free.lambda_tries and all(abs(k - cap) >= 3 for k in need):
            return cap
    raise AssertionError("no cap with clear decisions")


def test_a_pcg_cap_below_the_first_solve_costs_lambda_tries():
    nodes, pri, bt = lap_graph()
    cap = pick_pcg_cap(nodes, pri, bt)
    free, capped = pgg.PoseGraph(nodes, pri, bt), pgg.PoseGraph(nodes, pri, bt, cg_cap=cap)
    assert free.optimize() and capped.optimize()
    assert capped.accepted[0] == 0 and capped.lambda_tries > free.lambda_tries


def test_pcg_restatement_solves_the_damped_system():
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    nodes, pri, bt = lap_graph()
    g = pgg.PoseGraph(nodes, pri, bt)
    A, b = g._linearize(g.nodes, g.pri, g.btw)
    x, it, rel, trunc = pgg.pcg(A, b, 1e-5)
    xd = spla.spsolve((A + sp.diags(1e-5 * A.diagonal())).tocsc(), b)
    assert not trunc and rel <= 1e-10 and 0 < it < 4 * 400 + 200
    assert np.abs(x - xd).max() < 1e-7 * np.abs(xd).max()


# ---- long chains: the PCG's margin below its cap ------------------------------------------------------------------------------------------------
LONG = [(120, 0, "simple"), (120, 0, "graph"), (120, 1, "simple"), (120, 1, "graph"), (500, 0, "simple"), (500, 2, "simple"), (500, 2, "graph"),
        (1000, 1, "simple"), (1000, 1, "graph"), (5000, 1, "graph")]


def _first_and_smallest_lambda_systems(n, loops, weights):
    nodes, pri, bt = long_chain(n, loops, SIMPLE if weights == "simple" else GRAPH)
    g = pgg.PoseGraph(nodes, pri, bt)
    seen = {}

    def keep(A, b, lam):
        seen.setdefault("first", (A, b, lam))
        if "min" not in seen or lam < seen["min"][2]:
            seen["min"] = (A, b, lam)
    g.optimize(on_solve=keep)
    return g, seen


def test_long_chain_without_loops_under_graph_slam_weights_reaches_the_cap():
    """a 500-node chain pulled by a GraphSlam2D prior (sigma 0.01 against chain sigmas 0.25 / 0.15) with no loop: at the smallest lambda the
    oracle reaches (1.4e-8) the restated PCG stops at its cap of 2 200 iterations above the tolerance: this graph has no margin.  The
    device's sums round differently and its solves there stay below the cap (the GPU part); one that reached it would be rejected and
    lambda raised instead of taking the truncated step."""
    g, seen = _first_and_smallest_lambda_systems(500, 0, "graph")
    A, b, lam = seen["min"]
    assert lam < 1e-7
    _, it, rel, trunc = pgg.pcg(A, b, lam)
    assert trunc and it == 4 * 500 + 200 and rel > 1e-10


@pytest.mark.parametrize("n,loops,weights", LONG)
def test_long_chain_pcg_stays_below_its_cap(n, loops, weights):
    """the PCG iterations of the first damped system (lambda = 1e-5) and of the one at the smallest lambda the oracle reaches stay 10 %
    below 4 n + 200; a solve that reached the cap would be rejected (a wasted lambda try) rather than give a truncated step.  The 20 000-node
    chains are left to the GPU part: the LM restatement alone needs 100 sparse LU solves there."""
    w = SIMPLE if weights == "simple" else GRAPH
    nodes, pri, bt = long_chain(n, loops, w)
    g = pgg.PoseGraph(nodes, pri, bt)
    seen = {}

    def keep(A, b, lam):
        seen.setdefault("first", (A, b, lam))
        if "min" not in seen or lam < seen["min"][2]:
            seen["min"] = (A, b, lam)
    assert g.optimize(on_solve=keep) and g.status == 0
    cap = 4 * n + 200
    for key in ("first", "min"):
        A, b, lam = seen[key]
        _, it, rel, trunc = pgg.pcg(A, b, lam)
        assert not trunc and rel <= 1e-10 and it <= 0.9 * cap, (key, lam, it, cap)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------------------
def _api_factors(api, pri, bt):
    conv = lambda l: api.huber_loss(l[1]) if l[1] > 0 else api.diagonal_loss(1.0 / np.asarray(l[0]))
    return [(i, m, conv(l)) for i, m, l in pri], [(a, b, m, conv(l)) for a, b, m, l in bt]


def device_twice(api, nodes, pri, bt):
    p, b = _api_factors(api, pri, bt)
    r1 = api.pgo_optimize_graph(nodes, p, b)
    r2 = api.pgo_optimize_graph(nodes, p, b)
    keys = ("iterations", "lambda_tries", "cg_iterations", "initial_error", "final_error")
    assert r1[0] == r2[0] and r1[3] == r2[3] and [r1[2][k] for k in keys] == [r2[2][k] for k in keys]
    assert (r1[1] == r2[1]).all()
    return r1


NOISE = 1e-9   # relative: the device's fixed-order error sums are held to the oracle's within this (the initial error in compare)
# The device's CG iterations against pcg()'s: the sums are reduced in another order, so near convergence a solve can take a few more or
# fewer iterations.  Measured on an H100: 2 apart over 18 solves of a 5 000-node chain, 98 over 13 solves of a 1 000-node chain.
CG_SLACK_REL, CG_SLACK_PER_SOLVE = 0.01, 3


def compare(api, nodes, pri, bt, cg_cap=None, tol=1e-6, emulate_cg=True):
    """the device against the oracle, which runs the device's PCG rule (cap 4 n + 200 unless given): status, LM iterations, the accepted
    sequence and lambda tries, the initial error to 1e-9 relative, the device's CG iterations against the sum of pcg()'s, and the nodes to
    `tol` (theta wrapped) on SUCCESS.  emulate_cg=False runs the oracle with its direct solve only (no CG counts, no cap rule).  Otherwise the returned nodes must be the input (the C ABI writes them only on SUCCESS).

    One split is allowed, and returned as the index of the first try where the accepted flags differ: a try whose nonlinear decrease is
    within NOISE of the error is decided by the rounding of the two error sums, not by the step.  It must fall in the last LM iteration,
    so both runs end there with the same status; the tries after it may differ in number."""
    n = len(nodes)
    o = pgg.PoseGraph(nodes, pri, bt, cg_cap=(4 * n + 200 if cg_cap is None else cg_cap) if emulate_cg else None)
    o.optimize()
    st, x, rep, acc = device_twice(api, nodes, pri, bt)
    assert abs(rep["initial_error"] - o.errors[0]) <= NOISE * o.errors[0]
    assert (st, rep["iterations"]) == (o.status, o.iterations)
    split = next((k for k, (a, b) in enumerate(zip(acc, o.accepted)) if a != b), None)
    if split is None:
        assert acc == o.accepted and rep["lambda_tries"] == o.lambda_tries
        if emulate_cg:
            slack = CG_SLACK_REL * sum(o.cg_iterations) + CG_SLACK_PER_SOLVE * len(acc)
            assert abs(rep["cg_iterations"] - sum(o.cg_iterations)) <= slack, (rep["cg_iterations"], o.cg_iterations)
    else:
        d = o.decreases[split]
        assert d is not None and abs(d[0]) <= NOISE * d[1], (split, d)
        assert o.try_iterations[split] == o.iterations - 1, split
    if o.status == 0:
        assert np.abs(wrap(x - o.nodes_xyr())).max() < tol
    else:
        assert (x == np.asarray(nodes, float)).all()
    o.split = split
    return o, rep


@pytest.mark.gpu
@pytest.mark.parametrize("at", [0, 200, 400])
def test_device_unreferenced_node_is_a_zero_pivot(gpu_api, at):
    """one node that no factor references -- first, in the middle, last: ten rejected tries, ERROR_INCREASE, nodes untouched"""
    nodes, pri, bt = with_unreferenced_node(*lap_graph(), at=at)
    o, rep = compare(gpu_api, nodes, pri, bt)
    assert (o.status, o.iterations, o.lambda_tries) == (2, 1, 10)


@pytest.mark.gpu
def test_device_refuses_self_loops_and_accepts_duplicate_and_reversed_loop_edges(gpu_api):
    nodes, pri, bt = lap_graph()
    with pytest.raises(gpu_api.LamaError) as e:
        gpu_api.pgo_optimize_graph(nodes, *_api_factors(gpu_api, pri, bt + [(17, 17, [0.0, 0.0, 0.1], SIMPLE["loop"])]))
    assert e.value.code == -1
    from iris_lama_b200 import synth
    _, sn, se = synth.make_pose_graph(400, 300, seed=3)
    with pytest.raises(gpu_api.LamaError) as e:
        gpu_api.SimplePGO(sn, se + [(9, 9, [0.0, 0.0, 0.0])]).optimize()
    assert e.value.code == -1
    loops = bt[399:]
    dup = [(a, b, m, l) for a, b, m, l in loops[:40]]
    rev = [(b, a, pg.to_xyr(pg.inv(pg.from_xyr(m)))[0], l) for a, b, m, l in loops[40:80]]
    o, _ = compare(gpu_api, nodes, pri, bt[:399] + dup + rev + loops[80:] + dup)
    assert o.status == 0


def corridor(n=300, seed=4):
    """a corridor driven out along +x and back along -x: loop edges between node i and node n-1-i measure a rotation near pi"""
    rng = np.random.default_rng(seed)
    half = n // 2
    x = np.concatenate([np.arange(half) * 0.2, (half - 1) * 0.2 - np.arange(n - half) * 0.2])
    y = np.concatenate([np.zeros(half), np.full(n - half, 0.5)])
    th = np.concatenate([np.zeros(half), np.full(n - half, PI)])
    th[half + 1::3] = -PI                                                                   # the same heading, written as -pi
    truth = np.stack([x, y, th], 1)
    Xt = pg.from_xyr(truth)
    rel = pg.to_xyr(pg.mul(pg.inv(Xt[:-1]), Xt[1:])) + rng.normal(0, [0.01, 0.01, 0.003], (n - 1, 3))
    Rel = pg.from_xyr(rel)
    X = np.zeros((n, 4)); X[0] = Xt[0]
    for i in range(n - 1):
        X[i + 1] = pg.mul(X[i:i + 1], Rel[i:i + 1])[0]
    nodes = pg.to_xyr(X)
    nodes[half::4, 2] = np.where(nodes[half::4, 2] > 0, PI, -PI)                            # nodes at headings of exactly +-pi
    bt = [(i, i + 1, rel[i], SIMPLE["chain"]) for i in range(n - 1)]
    for i in range(5, half - 5, 7):
        j = n - 1 - i
        bt.append((i, j, pg.to_xyr(pg.mul(pg.inv(Xt[i:i + 1]), Xt[j:j + 1]))[0] + rng.normal(0, [0.01, 0.01, 0.002]), SIMPLE["loop"]))
    return nodes, [(0, nodes[0], SIMPLE["prior"])], bt


@pytest.mark.gpu
def test_device_heading_wrap_in_an_out_and_back_corridor(gpu_api):
    """node headings are converted to (cos, sin) on the host (se2_from_xyr in capi.cpp, the host libm's sin / cos) and back with the host's
    atan2; the error rotations near pi are taken on the device (se2_log: CUDA's atan2 of the s that se2_mul rounds without FMA)"""
    nodes, pri, bt = corridor()
    o, _ = compare(gpu_api, nodes, pri, bt)
    assert o.status == 0


def exact_pi_pair():
    """headings (t1, t2) whose fp64 states are exact negatives, so that v1^-1 v2 = (-1, +0): s = c1 (-s1) - s1 (-c1) = +0 exactly"""
    for k in range(1, 4000):
        t1 = 0.37 + k * 1e-3
        for t2 in (t1 - PI, _NA(t1 - PI, 0), _NA(t1 - PI, -10)):
            A, B = pg.from_xyr([0, 0, t1])[0], pg.from_xyr([0, 0, t2])[0]
            if B[0] == -A[0] and B[1] == -A[1]:
                return t1, float(t2)
    raise AssertionError("no pair")


def test_exact_pi_pair_is_exact_in_the_oracle_and_the_host_build(emu):
    t1, t2 = exact_pi_pair()
    A, B = pg.from_xyr([0, 0, t1]), pg.from_xyr([0, 0, t2])
    assert (emu(3, [0, 0, t1]) == A[0]).all() and (emu(3, [0, 0, t2]) == B[0]).all()   # the host libm agrees with numpy here
    D = pg.mul(pg.inv(A), B)
    assert D[0, 0] == -1.0 and D[0, 1] == 0.0 and math.copysign(1.0, D[0, 1]) == 1.0
    assert pg.log(D)[0, 2] == PI


@pytest.mark.gpu
def test_device_loop_error_rotation_of_exactly_pi(gpu_api):
    """a loop edge measured as the identity between two nodes whose states are exact negatives: the error rotation is (-1, +0), and
    atan2(+0, -1) = +pi decides the direction on the device (se2_mul rounds each product, so the cross terms cancel to +0) and in the oracle"""
    t1, t2 = exact_pi_pair()
    nodes, pri, bt = lap_graph()
    nodes = nodes.copy()
    nodes[50, 2], nodes[120, 2] = t1, t2
    X = pg.from_xyr(nodes)
    chain = pg.to_xyr(pg.mul(pg.inv(X[:-1]), X[1:]))
    bt = [(i, i + 1, chain[i], l) for i, (_, _, _, l) in enumerate(bt[:399])] + bt[399:] + [(50, 120, [0.0, 0.0, 0.0], pgg.huber(0.5))]
    E = pg.mul(pg.inv(pg.from_xyr([0.0, 0.0, 0.0])), pg.mul(pg.inv(X[50:51]), X[120:121]))
    assert E[0, 0] == -1.0 and E[0, 1] == 0.0 and pg.log(E)[0, 2] == PI
    compare(gpu_api, nodes, [(0, nodes[0], SIMPLE["prior"])], bt)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [1e3, 1e4, 1e5])
def test_device_far_off_coordinates(gpu_api, offset):
    """the lap graph translated by (offset, -offset): the oracle's translated and untranslated solutions differ by at most 1.7e-9 m at 1e5 m
    (measured), so the device is held to the usual 1e-6 against the oracle at the same offset"""
    nodes, pri, bt = lap_graph(offset=(offset, -offset))
    o, _ = compare(gpu_api, nodes, pri, bt)
    assert o.status == 0


def tiny_cases():
    rng = np.random.default_rng(12)
    P = SIMPLE["prior"]
    one = np.array([[1.0, 2.0, 0.3]])
    two = np.array([[0.0, 0.0, 0.0], [1.0, 0.2, 0.1]])
    five = np.cumsum(rng.uniform(-0.5, 0.5, (5, 3)), 0)
    X5 = pg.from_xyr(five)
    ch5 = pg.to_xyr(pg.mul(pg.inv(X5[:-1]), X5[1:]))
    return {
        "n1_prior": (one, [(0, [1.1, 1.9, 0.35], P)], []),
        "n2": (two, [(0, [0.05, 0.0, 0.0], P)], [(0, 1, [0.9, 0.1, 0.05], SIMPLE["chain"])]),
        "priors_only": (five, [(i, five[i] + [0.1, -0.1, 0.02], P) for i in range(5)], []),
        "two_priors_one_node": (two, [(0, [0.1, 0, 0], P), (0, [-0.1, 0.05, 0.02], pgg.diagonal([0.2, 0.3, 0.1]))],
                                [(0, 1, [0.9, 0.1, 0.05], SIMPLE["chain"])]),
        "all_fixed": (five, [(i, five[i] + [0.05, 0.0, 0.01], pgg.diagonal([0.1, 0.1, 0.1])) for i in range(5)],
                      [(i, i + 1, ch5[i], SIMPLE["chain"]) for i in range(4)]),
        "fixed_conflicts_with_odometry": (five, [(0, five[0], pgg.diagonal([0.1] * 3)), (4, five[4] + [2.0, -1.0, 0.4], pgg.diagonal([0.1] * 3))],
                                          [(i, i + 1, ch5[i], SIMPLE["chain"]) for i in range(4)]),
        "huber_prior": (five, [(0, five[0] + [0.5, 0.0, 0.1], pgg.huber(0.2))], [(i, i + 1, ch5[i], SIMPLE["chain"]) for i in range(4)]),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(tiny_cases()))
def test_device_tiny_and_odd_graphs(gpu_api, name):
    nodes, pri, bt = tiny_cases()[name]
    compare(gpu_api, nodes, pri, bt)


@pytest.mark.gpu
def test_device_simple_pgo_with_every_node_fixed_and_conflicting_fixed_poses(gpu_api):
    from iris_lama_b200 import synth
    truth, nodes, edges = synth.make_pose_graph(400, 300, seed=8)
    for fl in ([(i, truth[i]) for i in range(400)], [(0, truth[0]), (399, truth[399] + [1.0, -0.5, 0.3])]):
        o, g = pg.SimplePGO(nodes, edges, fl), gpu_api.SimplePGO(nodes, edges, fl)
        ok = o.optimize()
        assert g.optimize() == ok and ok
        assert (g.report["iterations"], g.report["lambda_tries"]) == (o.iterations, o.lambda_tries)
        assert np.abs(wrap(g.node_list - o.nodes_xyr())).max() < 1e-6


@pytest.mark.gpu
def test_device_huber_edges(gpu_api):
    """Huber weights: an edge whose error norm is exactly k at the start, k = 1e-9 on every factor (all in the linear branch), and a Huber
    prior.  At |e| = k both branches give the weight 1 (k / |e| = 1), so that case checks that the weight is continuous there; it cannot tell
    < from <= apart."""
    nodes, pri, bt = lap_graph()
    g = pgg.PoseGraph(nodes, pri, bt)
    _, rb, _, wb = g._errors(g.nodes, g.pri, g.btw)
    k = float(np.linalg.norm(rb[-1] / wb[-1]))
    assert k > 0
    at_k = bt[:-1] + [(bt[-1][0], bt[-1][1], bt[-1][2], pgg.huber(k))]
    ge = pgg.PoseGraph(nodes, pri, at_k)
    e_last = np.linalg.norm(pg.log(pg.mul(pg.inv(ge.btw[2][-1:]), pg.mul(pg.inv(ge.nodes[ge.btw[0][-1:]]), ge.nodes[ge.btw[1][-1:]]))))
    assert e_last == k                                         # exactly at k in the oracle; the device's norm may differ by an ulp
    compare(gpu_api, nodes, pri, at_k)
    compare(gpu_api, nodes, pri, [(a, b, m, pgg.huber(1e-9)) for a, b, m, _ in bt])
    compare(gpu_api, nodes, [(0, nodes[0] + [0.3, -0.2, 0.05], pgg.huber(0.1))], bt)


@pytest.mark.gpu
@pytest.mark.parametrize("n,loops,weights", LONG + [(500, 0, "graph"), (20000, 2, "graph")])
def test_device_long_chains(gpu_api, n, loops, weights, capsys):
    """long chains with few loops, the slow case of the PCG: the device follows the oracle; its CG iterations per solve are printed.

    * The 5 000-node chain under GraphSlam2D's weights splits at its 17th try (lambda = 4.6e6, last LM iteration): the oracle's decrease
      there is -1.1e-10 of an error of 2.48, below the rounding of the error sums, and the device accepts where the oracle goes on to
      lambda = 2.3e9 (DESIGN section 10).
    * The 500-node chain without loops under GraphSlam2D's weights sits at the cap: the restated PCG reaches its 2 200 iterations at the
      smallest lambda (see the CPU test), the device's stays below it (7 tries, all accepted).  It is compared with the oracle's direct
      solve, as is the 20 000-node chain, where restating the PCG on every try would take minutes on the CPU; there both stop at
      MAX_ITERATION after 100 iterations, each still lowering the error by ~3e-5 relative.
    * Left out: 20 000 nodes under SimplePGO's weights.  Its solves run close to the cap of 80 200 iterations (1.1e7 CG iterations over 166
      tries, 5.5 minutes on an H100), too long for the suite; 5 000 nodes under those weights is left out for the oracle's sake (its LM
      restatement takes 7 minutes on the CPU)."""
    nodes, pri, bt = long_chain(n, loops, SIMPLE if weights == "simple" else GRAPH)
    o, rep = compare(gpu_api, nodes, pri, bt, emulate_cg=(n, loops, weights) in LONG)
    if (n, loops, weights) == (5000, 1, "graph"):
        assert o.split == 16 and o.lambdas[16] == pytest.approx(4.58e6, rel=1e-3) and o.lambda_tries == 18
    else:
        assert o.split is None
    if (n, loops, weights) == (500, 0, "graph"):
        assert o.accepted == [1] * 7 and rep["cg_iterations"] < 7 * (4 * n + 200)
    assert o.status == (1 if n == 20000 else 0)
    with capsys.disabled():
        print(f"\n[pgo long chain] n={n} loops={loops} {weights}: {rep['cg_iterations'] / rep['lambda_tries']:.0f} CG iterations per solve, "
              f"{rep['lambda_tries']:.0f} solves, cap {4 * n + 200}")


@pytest.mark.gpu
def test_device_pcg_cap(gpu_api, monkeypatch):
    """LAMA_PGO_CG_MAX lowers the cap: at 1 every solve is truncated -- ten rejected tries, ERROR_INCREASE, nodes untouched; just below
    what the first solve needs, the LM takes the extra lambda tries that the oracle predicts with the same rule"""
    nodes, pri, bt = lap_graph()
    monkeypatch.setenv("LAMA_PGO_CG_MAX", "1")
    o, _ = compare(gpu_api, nodes, pri, bt, cg_cap=1)
    assert (o.status, o.lambda_tries) == (2, 10)
    cap = pick_pcg_cap(nodes, pri, bt)
    free = pgg.PoseGraph(nodes, pri, bt)
    free.optimize()
    monkeypatch.setenv("LAMA_PGO_CG_MAX", str(cap))
    o2, _ = compare(gpu_api, nodes, pri, bt, cg_cap=cap)
    assert o2.lambda_tries > free.lambda_tries and 0 in o2.accepted
