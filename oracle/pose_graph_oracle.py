"""CPU restatement of a miniSAM factor graph of PriorFactor<SE2> / BetweenFactor<SE2> whose factors carry a DiagonalLoss or a HuberLoss
(vendor/minisam/minisam: core/LossFunction.cpp:95-114, :190-203, LossFunction.h:199-202), optimised by LevenbergMarquardtOptimizer::optimize
(nonlinear/LevenbergMarquardtOptimizer.cpp:56-332 inside NonlinearOptimizer::optimize, nonlinear/NonlinearOptimizer.cpp:109-238): the graph
GraphSlam2D builds (src/graph_slam2d.cpp:209-226, :266-268, :394-430) and, with diagonal losses only, SimplePGO's.

TEST INFRASTRUCTURE ONLY (numpy + scipy): imported by tests/ and nothing else.  The SE2 arithmetic is pgo_oracle's; the linearisation and the
LM loop are pgo_oracle.SimplePGO's with the loss weights of each factor applied in place of its fixed 1 / sigma.  A test pins that SimplePGO's
graph given to PoseGraph reproduces pgo_oracle.SimplePGO bit for bit.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle.pgo_oracle import adj, exp, from_xyr, inv, log, mul, to_xyr


def loss_weights(e, w, k):
    """Row weights of each factor's loss at the errors e (n x 3): DiagonalLoss (core/LossFunction.cpp:95-114) scales row r by w_r = 1 / sigma_r;
    where k > 0, HuberLoss::Huber(k) (:190-203) scales every row by sqrt(weight(|e|)), weight = 1 if |e| < k else k / |e| (LossFunction.h:199-202)"""
    nrm = np.sqrt(e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1] + e[:, 2] * e[:, 2])
    hub = k > 0
    sw = np.sqrt(np.where(nrm < np.where(hub, k, 0.0), 1.0, np.where(hub, k, 1.0) / np.where(hub, np.abs(nrm), 1.0)))
    return np.where(hub[:, None], sw[:, None], w)


def diagonal(sigmas):
    """the (w, k) of DiagonalLoss::Sigmas(sigmas)"""
    return 1.0 / np.asarray(sigmas, float), 0.0


def huber(k):
    """the (w, k) of HuberLoss::Huber(k)"""
    return np.ones(3), float(k)


def pcg(A, b, lam, tol=1e-10, cap=None):
    """k_pgo_pcg restated: block-Jacobi preconditioned conjugate gradient on (A + lam diag(A)) x = b from x = 0, stopping when
    |r|^2 <= tol^2 |b|^2 or after `cap` iterations (default 4 n + 200).  Returns (x, iterations, |r| / |b|, truncated), truncated meaning
    the cap was reached above the tolerance; (None, 0, nan, False) when a damped diagonal entry is zero (the device solves nothing then)."""
    n = A.shape[0] // 3
    cap = 4 * n + 200 if cap is None else cap
    d = A.diagonal()
    if (d + lam * d == 0).any():
        return None, 0, float("nan"), False
    Ad = (A + sp.diags(lam * d)).tocsr()
    C = Ad.tocoo()
    on = C.row // 3 == C.col // 3
    blk = np.zeros((n, 3, 3))
    np.add.at(blk, (C.row[on] // 3, C.row[on] % 3, C.col[on] % 3), C.data[on])
    Minv = np.linalg.inv(blk)
    x = np.zeros_like(b)
    r = b.copy()
    z = np.einsum("nij,nj->ni", Minv, r.reshape(-1, 3)).ravel()
    p = z.copy()
    rz, bb = float(z @ r), float(b @ b)
    rr, it = bb, 0
    while it < cap and rr > tol * tol * bb and bb > 0.0:
        Ap = Ad @ p
        alpha = rz / float(p @ Ap)
        x += alpha * p
        r -= alpha * Ap
        rr = float(r @ r)
        z = np.einsum("nij,nj->ni", Minv, r.reshape(-1, 3)).ravel()
        rz2 = float(z @ r)
        p = z + (rz2 / rz) * p
        rz = rz2
        it += 1
    return x, it, (np.sqrt(rr / bb) if bb > 0 else 0.0), bool(it >= cap and rr > tol * tol * bb)


def _states(meas):
    """measured poses given as xyr triples or as SE2 states (cos, sin, tx, ty), which are taken as they are"""
    if not meas:
        return np.zeros((0, 4))
    return np.array([m if len(m) == 4 else from_xyr(m)[0] for m in meas], float)


class PoseGraph:
    """miniSAM FactorGraph of PriorFactor<SE2> / BetweenFactor<SE2>, each with a DiagonalLoss or a HuberLoss, optimised by
    LevenbergMarquardtOptimizer::optimize.  nodes: n x 3 xyr; priors [(node, meas, (w, k))]; betweens [(from, to, meas, (w, k))], in graph.add order
    (priors first).  After optimize(): status (0 SUCCESS, 1 MAX_ITERATION, 2 ERROR_INCREASE), iterations, lambda_tries, errors (0.5 errorSquaredNorm
    per accepted step), accepted (1 / 0 per lambda try), lambdas (lambda per try), try_iterations (the LM iteration of each try), decreases
    ((last error - trial error, last error) per try, None where no step was solved), and nodes (updated only on SUCCESS).

    A try whose damped system has a zero diagonal entry (a node no factor references) is rejected and lambda raised, as the reference does
    when its LDL^T reports RANK_DEFICIENCY.  With cg_cap set, every try also runs pcg() with that cap, cg_iterations records its iterations,
    and a solve truncated at the cap is rejected the same way (the device's rule); the step itself is the direct solve either way."""

    # LevenbergMarquardtOptimizerParams / NonlinearOptimizerParams defaults
    LAMBDA_INIT, INC_INIT, INC_UPDATE, DEC_MIN, LAMBDA_MIN, LAMBDA_MAX, GAIN_THRESH = 1e-5, 2.0, 2.0, 1.0 / 3.0, 1e-20, 1e10, 1e-3
    MAX_ITER, MIN_REL, MIN_ABS = 100, 1e-5, 1e-5

    def __init__(self, nodes_xyr, priors=(), betweens=(), cg_cap=None):
        self.nodes = from_xyr(nodes_xyr)
        pr = list(priors)
        bt = list(betweens)
        if any(b[0] == b[1] for b in bt):
            raise ValueError("a between factor needs two distinct nodes (from == to)")   # miniSAM's Hessian assembly assumes distinct keys
        self.cg_cap = cg_cap
        self.cg_iterations = []
        self.lambdas = []
        self.pri = (np.array([p[0] for p in pr], int), _states([p[1] for p in pr]),
                    np.array([p[2][0] for p in pr], float).reshape(-1, 3), np.array([p[2][1] for p in pr], float))
        self.btw = (np.array([b[0] for b in bt], int), np.array([b[1] for b in bt], int), _states([b[2] for b in bt]),
                    np.array([b[3][0] for b in bt], float).reshape(-1, 3), np.array([b[3][1] for b in bt], float))
        self.iterations = 0
        self.lambda_tries = 0
        self.errors = []
        self.accepted = []
        self.status = -1

    @staticmethod
    def _errors(X, pri, btw):
        """whitened errors and the loss row weights they were whitened with"""
        pr_idx, pr_meas, pr_w, pr_k = pri
        bt_i, bt_j, bt_meas, bt_w, bt_k = btw
        ep = log(mul(inv(pr_meas), X[pr_idx])) if len(pr_idx) else np.zeros((0, 3))      # PriorFactor::error
        eb = log(mul(inv(bt_meas), mul(inv(X[bt_i]), X[bt_j]))) if len(bt_i) else np.zeros((0, 3))   # BetweenFactor::error
        wp, wb = loss_weights(ep, pr_w, pr_k), loss_weights(eb, bt_w, bt_k)
        return ep * wp, eb * wb, wp, wb

    @classmethod
    def _err2(cls, X, pri, btw):
        rp, rb, _, _ = cls._errors(X, pri, btw)
        return 0.5 * (float((rp * rp).sum()) + float((rb * rb).sum()))

    def _linearize(self, X, pri, btw):
        """lower Hessian A = J^T J and b = -J^T r (linearization.cpp:150-230) as a full symmetric CSC matrix"""
        pr_idx = pri[0]
        bt_i, bt_j = btw[0], btw[1]
        n = len(X)
        rp, rb, wp, wb = self._errors(X, pri, btw)
        # BetweenFactor::jacobians: {Hcmp1 * Hinv, Hcmp2} = {Adj(v2^-1) * (-Adj(v1)), I}; rows scaled by the loss
        J1 = np.einsum("nij,njk->nik", adj(inv(X[bt_j])), -adj(X[bt_i])) * wb[:, :, None]
        J2 = np.eye(3)[None] * wb[:, :, None]
        Jp = np.eye(3)[None] * wp[:, :, None]
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

    def optimize(self, on_solve=None):
        """True on NonlinearOptimizationStatus::SUCCESS; node states updated in place then.  on_solve(A, b, lam), if given, sees the
        undamped system of every lambda try."""
        pri, btw = self.pri, self.btw
        X = self.nodes.copy()
        lam, inc = self.LAMBDA_INIT, self.INC_INIT
        last_err = self._err2(X, pri, btw)                                   # NonlinearOptimizer.cpp:175
        self.errors = [last_err]
        self.accepted = []
        self.lambdas = []
        self.cg_iterations = []
        self.decreases = []
        self.try_iterations = []
        self.iterations = 0
        self.status = 1                                                      # MAX_ITERATION unless decided otherwise
        while self.iterations < self.MAX_ITER:
            A, b = self._linearize(X, pri, btw)                              # LevenbergMarquardtOptimizer::iterate
            diag = A.diagonal().copy()
            ok = False
            while lam < self.LAMBDA_MAX:                                     # :121-151
                self.lambda_tries += 1
                self.lambdas.append(lam)
                self.try_iterations.append(self.iterations)
                self.decreases.append(None)
                if on_solve is not None:
                    on_solve(A, b, lam)
                truncated = False
                if self.cg_cap is not None:
                    _, it, _, truncated = pcg(A, b, lam, cap=self.cg_cap)
                    self.cg_iterations.append(it)
                if (diag + lam * diag == 0).any() or truncated:              # RANK_DEFICIENCY (SparseCholesky.cpp:26-31): no step (:139-144, :198-204)
                    self.accepted.append(0)
                    lam *= inc
                    inc *= self.INC_UPDATE
                    continue
                Ad = (A + sp.diags(lam * diag)).tocsc()                      # dumpLinearSystem_, diagonal damping (:275-283, :369-374)
                dx = spla.spsolve(Ad, b)
                Xn = mul(X, exp(dx.reshape(-1, 3)))                          # Variables::retract -> origin * exp(v) (Sophus.h:64-68)
                new_err = self._err2(Xn, pri, btw)
                nonlin = last_err - new_err                                  # values_curr_err = last_err_squared_norm_ (:115-116)
                self.decreases[-1] = (nonlin, last_err)
                lin = 0.5 * float(dx @ (lam * diag * dx + b))                # :241-247
                gain = nonlin / lin
                self.accepted.append(int(gain > self.GAIN_THRESH))
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
                self.status = 2
                return False                                                 # ERROR_INCREASE
            curr = new_err
            self.errors.append(curr)
            if curr - last_err > 1e-20:                                      # NonlinearOptimizer.cpp:213-216
                self.status = 2
                return False
            if (last_err - curr) < self.MIN_ABS or (last_err - curr) / last_err < self.MIN_REL:   # errorStopCondition_ :235-238
                self.nodes = X
                self.status = 0
                return True
            last_err = curr
        return False                                                         # MAX_ITERATION

    def nodes_xyr(self):
        return to_xyr(self.nodes)
