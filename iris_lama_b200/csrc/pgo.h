// pgo.h -- pose-graph optimisation on the device: lama::SimplePGO (SURVEY 8(f) row 3, BASELINE config 5) and GraphSlam2D's persistent
// graph (src/graph_slam2d.cpp:209-226, :266-268, :394-430), both through pgo_optimize_graph over an explicit factor list whose factors
// carry a DiagonalLoss or a HuberLoss.
//
// Reference: SimplePGO::optimize src/simple_pgo.cpp:48-105 -- a prior on node 0 (sigmas 1) or on the fixed nodes (sigmas 0.1),
// BetweenFactor<SE2> on consecutive nodes (measured = node[i]^-1 node[i+1]) and on the loop edges, all with sigmas (0.5, 0.5, 0.1),
// optimised by miniSAM's Levenberg-Marquardt (vendor/minisam/minisam/nonlinear/LevenbergMarquardtOptimizer.cpp:56-332, defaults .h:21-36,
// outer loop nonlinear/NonlinearOptimizer.cpp:109-238).  Factor arithmetic: slam/BetweenFactor.h:50-67, slam/PriorFactor.h:52-64,
// geometry/Sophus.h:45-74 (Local = log(origin^-1 t), Retract = origin exp(v), Jacobians -Adj / Adj(v2^-1) / I), whitening
// core/LossFunction.cpp:95-114, normal equations nonlinear/linearization.cpp:150-341 (b = -J^T r).
//
// What is different on the device: the damped normal equations (J^T J + lambda diag(J^T J)) dx = b are solved by a block-Jacobi
// preconditioned conjugate gradient running in ONE cooperative kernel (grid-wide barriers between the phases of an iteration, all
// reductions in a fixed order) instead of Eigen's SimplicialLDLT: the system is symmetric positive definite, so the solution is the
// same up to the CG tolerance (relative residual 1e-10), and the LM decisions (gain ratio, lambda schedule, stop rule) follow the
// reference line by line on the host in fp64.  Where the reference's LDL^T would report RANK_DEFICIENCY the device rejects the lambda try
// the same way (no step, lambda raised): a damped diagonal block with a zero diagonal entry (a node no factor references), and a PCG solve
// truncated at its iteration cap above the tolerance.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "lama_core.h"

namespace lama_b200 {

struct PgoEdge {
    int from, to;
    SE2 measured;
};
struct PgoFixed {
    int node;
    SE2 pose;
};
struct PgoReport {
    int status = -1;            // NonlinearOptimizationStatus: 0 SUCCESS, 1 MAX_ITERATION, 2 ERROR_INCREASE, 3 RANK_DEFICIENCY, 4 INVALID
    uint32_t iterations = 0;    // LM iterations (NonlinearOptimizer::iterations_)
    uint32_t lambda_tries = 0;  // tryLambda_ calls
    uint64_t cg_iterations = 0;
    double initial_error = 0, final_error = 0;
    double device_ms = 0;       // CUDA-event time of the whole optimisation
    std::vector<uint8_t> accepted;   // per tryLambda_ call in order: 1 the step was accepted, 0 rejected
};

// The loss of one factor: miniSAM's DiagonalLoss::Sigmas (core/LossFunction.cpp:95-114) when huber_k <= 0, else HuberLoss::Huber(huber_k)
// (:190-203, LossFunction.h:199-202) on the raw error: w = 1 if |e| < k else k / |e|, residual and Jacobians scaled by sqrt(w).
struct PgoLoss {
    double sigma[3] = {1, 1, 1};
    double huber_k  = 0;
};
struct PgoPrior {   // PriorFactor<SE2> (slam/PriorFactor.h:52-64)
    int node;
    SE2 measured;
    PgoLoss loss;
};
struct PgoBetween { // BetweenFactor<SE2> (slam/BetweenFactor.h:50-67): error = log(measured^-1 (x_from^-1 x_to))
    int from, to;
    SE2 measured;
    PgoLoss loss;
};

// miniSAM's LevenbergMarquardtOptimizer::optimize over an explicit factor graph (priors, then between factors, in graph.add order).
// On SUCCESS `nodes` holds the optimised poses; they are left untouched otherwise.  Returns a LAMA_* status (0 = the call worked; the
// optimiser's verdict is in report.status).
int pgo_optimize_graph(int device, std::vector<SE2>& nodes, const std::vector<PgoPrior>& priors, const std::vector<PgoBetween>& betweens, PgoReport& report,
                       std::string& err);

// SimplePGO::optimize: builds the reference's graph (simple_pgo.cpp:50-83) and runs pgo_optimize_graph.
int pgo_optimize(int device, std::vector<SE2>& nodes, const std::vector<PgoEdge>& edges, const std::vector<PgoFixed>& fixed, PgoReport& report, std::string& err);

}  // namespace lama_b200
