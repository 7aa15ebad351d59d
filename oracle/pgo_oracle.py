"""CPU restatement of lama::SimplePGO::optimize (src/simple_pgo.cpp:48-105) and of the miniSAM pieces it runs
(vendor/minisam/minisam): BetweenFactor / PriorFactor over Sophus SE2 (slam/BetweenFactor.h:50-67, slam/PriorFactor.h:52-64,
geometry/Sophus.h:45-74), DiagonalLoss whitening (core/LossFunction.cpp:95-114), lower-Hessian linearisation with b = -J^T r
(nonlinear/linearization.cpp:150-341), Levenberg-Marquardt with diagonal damping (nonlinear/LevenbergMarquardtOptimizer.cpp:56-332,
parameters .h:21-36) inside NonlinearOptimizer::optimize (nonlinear/NonlinearOptimizer.cpp:109-232, stop rule :235-238).

TEST INFRASTRUCTURE ONLY (numpy + scipy): imported by tests/ and nothing else.  **Parity unpinned**: the reference ships no
test or fixture for this path, and its linear solver (Eigen SimplicialLDLT with AMD ordering, linear/SparseCholesky.h:22-23) is
replaced by scipy's sparse LU -- the solution of the SPD system is unique, so the two agree to rounding (~1e-12 relative).
Independent pins in tests/test_pgo.py: the Jacobians against finite differences, a graph whose optimum is known in closed form.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

EPS = 1e-10   # SophusConstants<double>::epsilon (sophus.hpp:37-39)


# ---- Sophus SE2 on arrays of states (c, s, tx, ty) ----------------------------------------------------------------------------
def from_xyr(xyr):
    xyr = np.atleast_2d(np.asarray(xyr, float))
    c, s = np.cos(xyr[:, 2]), np.sin(xyr[:, 2])
    n = np.sqrt(c * c + s * s)                       # SO2(theta) normalises its unit complex (so2.hpp:100-103)
    return np.stack([c / n, s / n, xyr[:, 0], xyr[:, 1]], 1)


def to_xyr(X):
    X = np.atleast_2d(X)
    return np.stack([X[:, 2], X[:, 3], np.arctan2(X[:, 1], X[:, 0])], 1)


def mul(A, B):   # se2.hpp:153-157,262-265 ; so2.hpp:167-176,275-278 (product renormalised)
    c = A[:, 0] * B[:, 0] - A[:, 1] * B[:, 1]
    s = A[:, 0] * B[:, 1] + A[:, 1] * B[:, 0]
    n = np.sqrt(c * c + s * s)
    tx = A[:, 2] + (A[:, 0] * B[:, 2] - A[:, 1] * B[:, 3])
    ty = A[:, 3] + (A[:, 1] * B[:, 2] + A[:, 0] * B[:, 3])
    return np.stack([c / n, s / n, tx, ty], 1)


def inv(A):      # se2.hpp:163-167 ; so2.hpp:192-194
    c, s = A[:, 0], -A[:, 1]
    n = np.sqrt(c * c + s * s)
    c, s = c / n, s / n
    nx, ny = -A[:, 2], -A[:, 3]
    return np.stack([c, s, c * nx - s * ny, s * nx + c * ny], 1)


def exp(v):      # se2.hpp:389-412
    v = np.atleast_2d(v)
    th = v[:, 2]
    c, s = np.cos(th), np.sin(th)
    n = np.sqrt(c * c + s * s)
    c, s = c / n, s / n
    small = np.abs(th) < EPS
    ths = np.where(small, 1.0, th)
    a = np.where(small, 1.0 - th * th / 6.0, s / ths)
    b = np.where(small, 0.5 * th - th * th * th / 24.0, (1.0 - c) / ths)
    return np.stack([c, s, a * v[:, 0] - b * v[:, 1], b * v[:, 0] + a * v[:, 1]], 1)


def log(A):      # se2.hpp:519-542
    th = np.arctan2(A[:, 1], A[:, 0])
    half = 0.5 * th
    rm1 = A[:, 0] - 1.0
    small = np.abs(rm1) < EPS
    h = np.where(small, 1.0 - th * th / 12.0, -(half * A[:, 1]) / np.where(small, 1.0, rm1))
    return np.stack([h * A[:, 2] + half * A[:, 3], -half * A[:, 2] + h * A[:, 3], th], 1)


def adj(A):      # se2.hpp:125-133
    M = np.zeros((len(A), 3, 3))
    M[:, 0, 0] = A[:, 0]; M[:, 0, 1] = -A[:, 1]; M[:, 1, 0] = A[:, 1]; M[:, 1, 1] = A[:, 0]
    M[:, 0, 2] = A[:, 3]; M[:, 1, 2] = -A[:, 2]; M[:, 2, 2] = 1.0
    return M


class SimplePGO:
    """lama::SimplePGO (include/lama/simple_pgo.h:43-57): node_list, edge_list = [(from, to, xyr)], fixed_list = [(index, xyr)]"""

    # LevenbergMarquardtOptimizerParams / NonlinearOptimizerParams defaults
    LAMBDA_INIT, INC_INIT, INC_UPDATE, DEC_MIN, LAMBDA_MIN, LAMBDA_MAX, GAIN_THRESH = 1e-5, 2.0, 2.0, 1.0 / 3.0, 1e-20, 1e10, 1e-3
    MAX_ITER, MIN_REL, MIN_ABS = 100, 1e-5, 1e-5

    def __init__(self, nodes_xyr, edges=(), fixed=()):
        self.nodes = from_xyr(nodes_xyr)
        self.edges = list(edges)
        if any(e[0] == e[1] for e in self.edges):
            raise ValueError("an edge needs two distinct nodes (from == to)")   # miniSAM's Hessian assembly assumes distinct keys
        self.fixed = list(fixed)
        self.iterations = 0
        self.lambda_tries = 0
        self.errors = []

    def _factors(self):
        X = self.nodes
        n = len(X)
        # priors (simple_pgo.cpp:52-63)
        if not self.fixed:
            pr_idx, pr_meas, pr_w = np.array([0]), X[:1].copy(), np.full((1, 3), 1.0)
        else:
            pr_idx = np.array([i for i, _ in self.fixed])
            pr_meas = from_xyr([p for _, p in self.fixed])
            pr_w = np.full((len(self.fixed), 3), 1.0 / 0.1)
        # odometry chain (:66-73): diff = node[i] - node[i+1] = node[i]^-1 * node[i+1] (pose2d.cpp:81-84), sigmas (0.5, 0.5, 0.1); loop edges (:76-82)
        i0 = np.arange(n - 1)
        od_meas = mul(inv(X[i0]), X[i0 + 1])
        ef = np.array([e[0] for e in self.edges], int)
        et = np.array([e[1] for e in self.edges], int)
        bt_i = np.concatenate([i0, ef])
        bt_j = np.concatenate([i0 + 1, et])
        bt_meas = np.concatenate([od_meas, from_xyr([e[2] for e in self.edges])]) if self.edges else od_meas
        bt_w = np.tile(1.0 / np.array([0.5, 0.5, 0.1]), (len(bt_i), 1))
        return (pr_idx, pr_meas, pr_w), (bt_i, bt_j, bt_meas, bt_w)

    @staticmethod
    def _errors(X, pri, btw):
        pr_idx, pr_meas, pr_w = pri
        bt_i, bt_j, bt_meas, bt_w = btw
        rp = log(mul(inv(pr_meas), X[pr_idx])) * pr_w                                  # PriorFactor::error, whitened
        rb = log(mul(inv(bt_meas), mul(inv(X[bt_i]), X[bt_j]))) * bt_w                 # BetweenFactor::error, whitened
        return rp, rb

    @classmethod
    def _err2(cls, X, pri, btw):
        rp, rb = cls._errors(X, pri, btw)
        return 0.5 * (float((rp * rp).sum()) + float((rb * rb).sum()))

    def _linearize(self, X, pri, btw):
        """lower Hessian A = J^T J and b = -J^T r (linearization.cpp:150-230) as a full symmetric CSC matrix"""
        pr_idx, pr_meas, pr_w = pri
        bt_i, bt_j, bt_meas, bt_w = btw
        n = len(X)
        rp, rb = self._errors(X, pri, btw)
        # BetweenFactor::jacobians: {Hcmp1 * Hinv, Hcmp2} = {Adj(v2^-1) * (-Adj(v1)), I}; rows scaled by the loss
        J1 = np.einsum("nij,njk->nik", adj(inv(X[bt_j])), -adj(X[bt_i])) * bt_w[:, :, None]
        J2 = np.eye(3)[None] * bt_w[:, :, None]
        Jp = np.eye(3)[None] * pr_w[:, :, None]
        b = np.zeros((n, 3))
        np.add.at(b, pr_idx, -np.einsum("nji,nj->ni", Jp, rp))
        np.add.at(b, bt_i, -np.einsum("nji,nj->ni", J1, rb))
        np.add.at(b, bt_j, -np.einsum("nji,nj->ni", J2, rb))
        rows, cols, vals = [], [], []

        def block(bi, bj, M):
            r = (3 * bi)[:, None, None] + np.arange(3)[None, :, None] + np.zeros((1, 1, 3), int)
            c = (3 * bj)[:, None, None] + np.arange(3)[None, None, :] + np.zeros((1, 3, 1), int)
            rows.append(r.ravel()); cols.append(c.ravel()); vals.append(M.ravel())
        block(pr_idx, pr_idx, np.einsum("nki,nkj->nij", Jp, Jp))
        block(bt_i, bt_i, np.einsum("nki,nkj->nij", J1, J1))
        block(bt_j, bt_j, np.einsum("nki,nkj->nij", J2, J2))
        H12 = np.einsum("nki,nkj->nij", J1, J2)
        block(bt_i, bt_j, H12)
        block(bt_j, bt_i, np.transpose(H12, (0, 2, 1)))
        A = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * n, 3 * n)).tocsc()
        return A, b.ravel()

    def optimize(self):
        """SimplePGO::optimize: True on NonlinearOptimizationStatus::SUCCESS; node states updated in place then"""
        pri, btw = self._factors()
        X = self.nodes.copy()
        lam, inc = self.LAMBDA_INIT, self.INC_INIT
        last_err = self._err2(X, pri, btw)                                   # NonlinearOptimizer.cpp:175
        self.errors = [last_err]
        self.iterations = 0
        while self.iterations < self.MAX_ITER:
            A, b = self._linearize(X, pri, btw)                              # LevenbergMarquardtOptimizer::iterate
            diag = A.diagonal().copy()
            ok = False
            while lam < self.LAMBDA_MAX:                                     # :121-151
                self.lambda_tries += 1
                if (diag + lam * diag == 0).any():                           # zero pivot: RANK_DEFICIENCY (SparseCholesky.cpp:26-31), no step (:139-144)
                    lam *= inc
                    inc *= self.INC_UPDATE
                    continue
                Ad = (A + sp.diags(lam * diag)).tocsc()                      # dumpLinearSystem_, diagonal damping (:275-283, :369-374)
                dx = spla.spsolve(Ad, b)
                Xn = mul(X, exp(dx.reshape(-1, 3)))                          # Variables::retract -> origin * exp(v) (Sophus.h:64-68)
                new_err = self._err2(Xn, pri, btw)
                nonlin = last_err - new_err                                  # values_curr_err = last_err_squared_norm_ (:115-116)
                lin = 0.5 * float(dx @ (lam * diag * dx + b))                # :241-247
                gain = nonlin / lin
                if gain > self.GAIN_THRESH:                                  # :256-265
                    X = Xn
                    lam = max(self.LAMBDA_MIN, lam * max(self.DEC_MIN, 1.0 - (2.0 * gain - 1.0) ** 3))   # decreaseLambda_ :342-348
                    inc = self.INC_INIT
                    ok = True
                    break
                lam *= inc                                                   # increaseLambda_ :336-339
                inc *= self.INC_UPDATE
            self.iterations += 1
            if not ok:
                return False                                                 # ERROR_INCREASE
            curr = new_err
            self.errors.append(curr)
            if curr - last_err > 1e-20:                                      # NonlinearOptimizer.cpp:213-216
                return False
            if (last_err - curr) < self.MIN_ABS or (last_err - curr) / last_err < self.MIN_REL:   # errorStopCondition_ :235-238
                self.nodes = X
                return True
            last_err = curr
        return False                                                         # MAX_ITERATION

    def nodes_xyr(self):
        return to_xyr(self.nodes)
