// pgo.cu -- see pgo.h.  Kernels: k_pgo_linearize (per factor: loss weights, whitened error, Jacobian, Hessian blocks), k_pgo_assemble (per node: diagonal
// block and right-hand side, gathered in a fixed order: no atomics), k_pgo_pcg (cooperative: the whole damped solve), k_pgo_retract,
// k_pgo_error (fixed-order two-level sum of the whitened squared errors).
#include "pgo.h"

#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "cuda_owned.h"
#include "engine.h"   // status codes

namespace cg = cooperative_groups;

namespace lama_b200 {

namespace {

struct PgoView {
    int n_nodes, n_prior, n_between;
    // factors
    const int* prior_node;  const SE2* prior_meas;  const double* prior_w;  const double* prior_k;   // n_prior, n_prior, n_prior x 3, n_prior
    const int* bt_i;  const int* bt_j;  const SE2* bt_meas;  const double* bt_w;  const double* bt_k;   // n_between (x 3); w = 1 / sigma, k = Huber k (0: none)
    // adjacency of the nodes: adj[adj_ptr[i] .. adj_ptr[i + 1]) = factor << 2 | role (0: first key of a between factor, 1: second key, 2: prior)
    const int* adj_ptr;  const int* adj;
    // linearisation
    double* we_prior;  // n_prior x 3    row weights of the loss at the linearisation point (1 / sigma, or sqrt(Huber weight))
    double* we_bt;     // n_between x 3
    double* r_prior;   // n_prior x 3    whitened errors
    double* r_bt;      // n_between x 3
    double* J1;        // n_between x 9  whitened Jacobian wrt the first key (the second key's is diag(w))
    double* B;         // n_between x 9  off-diagonal Hessian block J1^T diag(w)
    double* D;         // n_nodes x 9    diagonal Hessian blocks
    double* b;         // n_nodes x 3    -J^T r
};

__device__ __forceinline__ void mat3_mul(const double* a, const double* b, double* c)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
}

// Row weights of a factor's loss at the error e: DiagonalLoss (core/LossFunction.cpp:95-114) scales row k by 1 / sigma_k; HuberLoss
// (:190-203) scales every row by sqrt(w), w = 1 if |e| < k else k / |e| (LossFunction.h:199-202), so the factor adds w |e|^2 to
// errorSquaredNorm.  The Huber weight depends on the point the error is taken at, so it is recomputed at every linearisation and trial point.
__device__ __forceinline__ void loss_weights(const double* w0, double k, const double e[3], double w[3])
{
    if (k > 0.0) {
        const double nrm = sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
        const double sw = sqrt(nrm < k ? 1.0 : k / fabs(nrm));
        w[0] = w[1] = w[2] = sw;
    } else {
        w[0] = w0[0]; w[1] = w0[1]; w[2] = w0[2];
    }
}

// BetweenFactor::error / jacobians (slam/BetweenFactor.h:50-67) and PriorFactor::error (slam/PriorFactor.h:52-56), whitened by the loss.
// with_jacobians: a linearisation, which also records the loss weights that k_pgo_assemble reads; otherwise only the errors (trial points).
__global__ void k_pgo_linearize(PgoView g, const SE2* __restrict__ X, int with_jacobians)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < g.n_between) {
        const SE2 v1 = X[g.bt_i[f]], v2 = X[g.bt_j[f]];
        const SE2 diff = se2_mul(se2_inv(v1), v2);                         // Compose(Inverse(v1), v2)
        double e[3], w[3];
        se2_log(se2_mul(se2_inv(g.bt_meas[f]), diff), e);                 // Local(diff_, diff) = log(diff_^-1 diff)  (Sophus.h:53-57)
        loss_weights(g.bt_w + 3 * (size_t)f, g.bt_k[f], e, w);
        for (int k = 0; k < 3; ++k) g.r_bt[3 * (size_t)f + k] = e[k] * w[k];
        if (with_jacobians) {
            for (int k = 0; k < 3; ++k) g.we_bt[3 * (size_t)f + k] = w[k];
            double a2[9], a1[9], j1[9];
            se2_adj(se2_inv(v2), a2);                                      // Hcmp1 = s2.inverse().Adj()  (Sophus.h:77-81)
            se2_adj(v1, a1);
            for (int k = 0; k < 9; ++k) a1[k] = -a1[k];                    // Hinv = -s.Adj()            (Sophus.h:73)
            mat3_mul(a2, a1, j1);                                          // Hcmp1 * Hinv
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) j1[r * 3 + c] *= w[r];         // rows scaled by the loss
            double* J = g.J1 + 9 * (size_t)f;
            double* Bf = g.B + 9 * (size_t)f;
            for (int k = 0; k < 9; ++k) J[k] = j1[k];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) Bf[r * 3 + c] = j1[c * 3 + r] * w[c];   // (J1^T J2)[r][c] = J1[c][r] * w[c]
        }
    }
    if (f < g.n_prior) {
        double e[3], w[3];
        se2_log(se2_mul(se2_inv(g.prior_meas[f]), X[g.prior_node[f]]), e);
        loss_weights(g.prior_w + 3 * (size_t)f, g.prior_k[f], e, w);
        for (int k = 0; k < 3; ++k) g.r_prior[3 * (size_t)f + k] = e[k] * w[k];
        if (with_jacobians)
            for (int k = 0; k < 3; ++k) g.we_prior[3 * (size_t)f + k] = w[k];
    }
}

// A = J^T J (block diagonal part) and b = -J^T r per node, contributions added in adjacency order (linearization.cpp:150-230)
__global__ void k_pgo_assemble(PgoView g)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.n_nodes) return;
    double d[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bb[3] = {0, 0, 0};
    for (int k = g.adj_ptr[i]; k < g.adj_ptr[i + 1]; ++k) {
        const int f = g.adj[k] >> 2, role = g.adj[k] & 3;
        if (role == 0) {
            const double* J = g.J1 + 9 * (size_t)f;
            const double* r = g.r_bt + 3 * (size_t)f;
            for (int a = 0; a < 3; ++a) {
                for (int c = 0; c < 3; ++c) d[a * 3 + c] += J[a] * J[c] + J[3 + a] * J[3 + c] + J[6 + a] * J[6 + c];
                bb[a] -= J[a] * r[0] + J[3 + a] * r[1] + J[6 + a] * r[2];
            }
        } else {
            const double* w = role == 1 ? g.we_bt + 3 * (size_t)f : g.we_prior + 3 * (size_t)f;   // the loss weights of this linearisation
            const double* r = role == 1 ? g.r_bt + 3 * (size_t)f : g.r_prior + 3 * (size_t)f;
            for (int a = 0; a < 3; ++a) {
                d[a * 4] += w[a] * w[a];
                bb[a] -= w[a] * r[a];
            }
        }
    }
    for (int k = 0; k < 9; ++k) g.D[9 * (size_t)i + k] = d[k];
    for (int k = 0; k < 3; ++k) g.b[3 * (size_t)i + k] = bb[k];
}

// ---- cooperative preconditioned conjugate gradient ------------------------------------------------------------------------------------
struct PcgBuffers {
    double* x;  double* r;  double* z;  double* p;  double* Ap;   // n_nodes x 3 each
    double* Minv;      // n_nodes x 9: inverse of the damped diagonal block
    double* partial;   // gridDim x 4 scratch of the reductions
    double* out;       // {r.r at exit, b.b, 0.5 dx.(lambda diag dx + b), iterations, damped diagonal blocks with a zero diagonal entry}
};

__device__ __forceinline__ double block_sum(double v, double* sh)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
    return t;
}
// grid-wide sum in a fixed order: block partials, grid barrier, every block adds the partials up in index order
__device__ __forceinline__ double grid_sum(cg::grid_group& grid, double v, double* sh, double* partial, int slot)
{
    const double bs = block_sum(v, sh);
    if (threadIdx.x == 0) partial[(size_t)blockIdx.x * 4 + slot] = bs;
    grid.sync();
    double t = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) t += __ldcg(partial + (size_t)b * 4 + slot);
    return t;
}

__global__ void __launch_bounds__(256)
k_pgo_pcg(PgoView g, PcgBuffers w, double lambda, double rel_tol, int max_iter)
{
    cg::grid_group grid = cg::this_grid();
    __shared__ double sh[8];
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthreads = gridDim.x * blockDim.x;
    const int n = g.n_nodes;
    // damped diagonal blocks and their inverses (block-Jacobi preconditioner); x = 0, r = b, z = M^-1 r, p = z
    double loc_rz = 0.0, loc_bb = 0.0, loc_zero = 0.0;
    for (int i = tid; i < n; i += nthreads) {
        double m[9];
        for (int k = 0; k < 9; ++k) m[k] = g.D[9 * (size_t)i + k];
        m[0] += lambda * m[0]; m[4] += lambda * m[4]; m[8] += lambda * m[8];   // updateDumpingHessianDiag (LevenbergMarquardtOptimizer.cpp:369-374)
        // a zero diagonal entry: a node no factor references (lambda * 0 = 0), where the reference's LDL^T meets a zero pivot
        if (m[0] == 0.0 || m[4] == 0.0 || m[8] == 0.0) loc_zero += 1.0;
        const double c0 = m[4] * m[8] - m[5] * m[7], c1 = m[5] * m[6] - m[3] * m[8], c2 = m[3] * m[7] - m[4] * m[6];
        const double det = m[0] * c0 + m[1] * c1 + m[2] * c2, id = 1.0 / det;
        double* mi = w.Minv + 9 * (size_t)i;
        mi[0] = c0 * id; mi[1] = (m[2] * m[7] - m[1] * m[8]) * id; mi[2] = (m[1] * m[5] - m[2] * m[4]) * id;
        mi[3] = c1 * id; mi[4] = (m[0] * m[8] - m[2] * m[6]) * id; mi[5] = (m[2] * m[3] - m[0] * m[5]) * id;
        mi[6] = c2 * id; mi[7] = (m[1] * m[6] - m[0] * m[7]) * id; mi[8] = (m[0] * m[4] - m[1] * m[3]) * id;
        for (int a = 0; a < 3; ++a) {
            const double ra = g.b[3 * (size_t)i + a];
            w.x[3 * (size_t)i + a] = 0.0;
            w.r[3 * (size_t)i + a] = ra;
            loc_bb += ra * ra;
        }
        for (int a = 0; a < 3; ++a) {
            const double za = mi[a * 3] * g.b[3 * (size_t)i] + mi[a * 3 + 1] * g.b[3 * (size_t)i + 1] + mi[a * 3 + 2] * g.b[3 * (size_t)i + 2];
            w.z[3 * (size_t)i + a] = za;
            w.p[3 * (size_t)i + a] = za;
            loc_rz += za * g.b[3 * (size_t)i + a];
        }
    }
    double rz = grid_sum(grid, loc_rz, sh, w.partial, 0);
    const double bb = grid_sum(grid, loc_bb, sh, w.partial, 1);
    const double zero_blocks = grid_sum(grid, loc_zero, sh, w.partial, 3);   // the factorisation failed: no solve, x stays 0
    double rr = bb;
    int it = 0;
    while (zero_blocks == 0.0 && it < max_iter && rr > rel_tol * rel_tol * bb && bb > 0.0) {
        // Ap = (D + lambda diag D) p + off-diagonal blocks, gathered per node in adjacency order
        double loc_pap = 0.0;
        for (int i = tid; i < n; i += nthreads) {
            const double* d = g.D + 9 * (size_t)i;
            const double p0 = __ldcg(w.p + 3 * (size_t)i), p1 = __ldcg(w.p + 3 * (size_t)i + 1), p2 = __ldcg(w.p + 3 * (size_t)i + 2);
            double a0 = d[0] * p0 + d[1] * p1 + d[2] * p2 + lambda * d[0] * p0;
            double a1 = d[3] * p0 + d[4] * p1 + d[5] * p2 + lambda * d[4] * p1;
            double a2 = d[6] * p0 + d[7] * p1 + d[8] * p2 + lambda * d[8] * p2;
            for (int k = g.adj_ptr[i]; k < g.adj_ptr[i + 1]; ++k) {
                const int f = g.adj[k] >> 2, role = g.adj[k] & 3;
                if (role == 2) continue;
                const double* Bf = g.B + 9 * (size_t)f;
                if (role == 0) {   // this node is the first key: + B p_j
                    const int j = g.bt_j[f];
                    const double q0 = __ldcg(w.p + 3 * (size_t)j), q1 = __ldcg(w.p + 3 * (size_t)j + 1), q2 = __ldcg(w.p + 3 * (size_t)j + 2);
                    a0 += Bf[0] * q0 + Bf[1] * q1 + Bf[2] * q2;
                    a1 += Bf[3] * q0 + Bf[4] * q1 + Bf[5] * q2;
                    a2 += Bf[6] * q0 + Bf[7] * q1 + Bf[8] * q2;
                } else {           // second key: + B^T p_i
                    const int j = g.bt_i[f];
                    const double q0 = __ldcg(w.p + 3 * (size_t)j), q1 = __ldcg(w.p + 3 * (size_t)j + 1), q2 = __ldcg(w.p + 3 * (size_t)j + 2);
                    a0 += Bf[0] * q0 + Bf[3] * q1 + Bf[6] * q2;
                    a1 += Bf[1] * q0 + Bf[4] * q1 + Bf[7] * q2;
                    a2 += Bf[2] * q0 + Bf[5] * q1 + Bf[8] * q2;
                }
            }
            w.Ap[3 * (size_t)i] = a0; w.Ap[3 * (size_t)i + 1] = a1; w.Ap[3 * (size_t)i + 2] = a2;
            loc_pap += p0 * a0 + p1 * a1 + p2 * a2;
        }
        const double pap = grid_sum(grid, loc_pap, sh, w.partial, 2);
        const double alpha = rz / pap;
        double loc_rr = 0.0, loc_rz2 = 0.0;
        for (int i = tid; i < n; i += nthreads) {
            double rn[3];
            for (int a = 0; a < 3; ++a) {
                const size_t k = 3 * (size_t)i + a;
                w.x[k] += alpha * w.p[k];
                rn[a] = w.r[k] - alpha * w.Ap[k];
                w.r[k] = rn[a];
                loc_rr += rn[a] * rn[a];
            }
            const double* mi = w.Minv + 9 * (size_t)i;
            for (int a = 0; a < 3; ++a) {
                const double za = mi[a * 3] * rn[0] + mi[a * 3 + 1] * rn[1] + mi[a * 3 + 2] * rn[2];
                w.z[3 * (size_t)i + a] = za;
                loc_rz2 += za * rn[a];
            }
        }
        rr = grid_sum(grid, loc_rr, sh, w.partial, 3);
        const double rz2 = grid_sum(grid, loc_rz2, sh, w.partial, 0);
        const double beta = rz2 / rz;
        rz = rz2;
        for (int i = tid; i < n; i += nthreads)
            for (int a = 0; a < 3; ++a) {
                const size_t k = 3 * (size_t)i + a;
                w.p[k] = w.z[k] + beta * w.p[k];
            }
        grid.sync();
        ++it;
    }
    // linear error improvement 0.5 dx . (lambda diag(A) dx + g), g = b  (LevenbergMarquardtOptimizer.cpp:241-247)
    double loc_lin = 0.0;
    for (int i = tid; i < n; i += nthreads)
        for (int a = 0; a < 3; ++a) {
            const size_t k = 3 * (size_t)i + a;
            const double dx = w.x[k];
            loc_lin += dx * (lambda * g.D[9 * (size_t)i + 4 * a] * dx + g.b[k]);
        }
    const double lin = grid_sum(grid, loc_lin, sh, w.partial, 1);
    if (tid == 0) {
        w.out[0] = rr;
        w.out[1] = bb;
        w.out[2] = 0.5 * lin;
        w.out[3] = (double)it;
        w.out[4] = zero_blocks;
    }
}

// Variables::retract: x <- x exp(dx)  (Sophus.h:64-68)
__global__ void k_pgo_retract(int n, const SE2* __restrict__ X, const double* __restrict__ dx, SE2* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double h[3] = {dx[3 * (size_t)i], dx[3 * (size_t)i + 1], dx[3 * (size_t)i + 2]};
    out[i] = se2_mul(X[i], se2_exp(h));
}

// 0.5 * FactorGraph::errorSquaredNorm: block partials in factor order, then one thread adds them up
__global__ void k_pgo_error_partial(PgoView g, double* __restrict__ partial)
{
    __shared__ double sh[8];
    double v = 0.0;
    const int nb3 = 3 * g.n_between, np3 = 3 * g.n_prior;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < nb3 + np3; k += gridDim.x * blockDim.x) {
        const double e = k < nb3 ? g.r_bt[k] : g.r_prior[k - nb3];
        v += e * e;
    }
    const double s = block_sum(v, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}
__global__ void k_pgo_error_final(const double* __restrict__ partial, int n, double* __restrict__ out)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < n; ++i) t += partial[i];
        *out = 0.5 * t;
    }
}

struct DeviceArena {   // the device arrays of one solve, freed together
    std::vector<DeviceArray<char>> blocks;
    template <typename T> T* alloc(size_t n, cudaError_t& e)
    {
        if (e != cudaSuccess) return nullptr;
        blocks.emplace_back();
        e = blocks.back().alloc(std::max<size_t>(n, 1) * sizeof(T));
        return (T*)blocks.back().get();
    }
    template <typename T> T* upload(const std::vector<T>& v, cudaError_t& e)
    {
        T* p = alloc<T>(v.size(), e);
        if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
        return p;
    }
};

}  // namespace

int pgo_optimize_graph(int device, std::vector<SE2>& nodes, const std::vector<PgoPrior>& priors, const std::vector<PgoBetween>& betweens, PgoReport& rep,
                       std::string& err)
{
    rep = PgoReport();
    const int n = (int)nodes.size();
    if (n < 1) { err = "pose graph: no nodes"; return LAMA_ERR_ARG; }
    if (priors.empty() && betweens.empty()) { err = "pose graph: no factors"; return LAMA_ERR_ARG; }
    auto bad_loss = [](const PgoLoss& l) {
        if (l.huber_k > 0.0) return !std::isfinite(l.huber_k);
        for (int k = 0; k < 3; ++k)
            if (!(l.sigma[k] > 0.0) || !std::isfinite(l.sigma[k])) return true;
        return false;
    };
    for (const PgoPrior& p : priors) {
        if (p.node < 0 || p.node >= n) { err = "pose graph: prior node out of range"; return LAMA_ERR_ARG; }
        if (bad_loss(p.loss)) { err = "pose graph: a prior's loss needs sigmas > 0 or a finite Huber k > 0"; return LAMA_ERR_ARG; }
    }
    for (const PgoBetween& e : betweens) {
        if (e.from < 0 || e.from >= n || e.to < 0 || e.to >= n) { err = "pose graph: between factor index out of range"; return LAMA_ERR_ARG; }
        if (e.from == e.to) { err = "pose graph: a between factor needs two distinct nodes (from == to)"; return LAMA_ERR_ARG; }
        if (bad_loss(e.loss)) { err = "pose graph: a between factor's loss needs sigmas > 0 or a finite Huber k > 0"; return LAMA_ERR_ARG; }
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return LAMA_ERR_NO_DEVICE; }
    if (cudaSetDevice(device) != cudaSuccess) { err = "invalid device index"; return LAMA_ERR_ARG; }

    const int nb = (int)betweens.size(), np = (int)priors.size();
    std::vector<int> prior_node((size_t)np), bt_i((size_t)nb), bt_j((size_t)nb);
    std::vector<SE2> prior_meas((size_t)np), bt_meas((size_t)nb);
    std::vector<double> prior_w((size_t)np * 3), prior_k((size_t)np), bt_w((size_t)nb * 3), bt_k((size_t)nb);
    for (int f = 0; f < np; ++f) {
        prior_node[(size_t)f] = priors[(size_t)f].node; prior_meas[(size_t)f] = priors[(size_t)f].measured;
        prior_k[(size_t)f] = std::max(0.0, priors[(size_t)f].loss.huber_k);
        for (int k = 0; k < 3; ++k) prior_w[(size_t)f * 3 + k] = 1.0 / priors[(size_t)f].loss.sigma[k];   // DiagonalLoss::Sigmas: cwiseInverse
    }
    for (int f = 0; f < nb; ++f) {
        const PgoBetween& e = betweens[(size_t)f];
        bt_i[(size_t)f] = e.from; bt_j[(size_t)f] = e.to; bt_meas[(size_t)f] = e.measured;
        bt_k[(size_t)f] = std::max(0.0, e.loss.huber_k);
        for (int k = 0; k < 3; ++k) bt_w[(size_t)f * 3 + k] = 1.0 / e.loss.sigma[k];
    }
    // adjacency in factor order (priors first, like graph.add's order)
    std::vector<int> deg((size_t)n + 1, 0);
    for (int f = 0; f < np; ++f) ++deg[(size_t)prior_node[f] + 1];
    for (int f = 0; f < nb; ++f) { ++deg[(size_t)bt_i[f] + 1]; ++deg[(size_t)bt_j[f] + 1]; }
    std::vector<int> adj_ptr((size_t)n + 1, 0);
    for (int i = 0; i < n; ++i) adj_ptr[(size_t)i + 1] = adj_ptr[(size_t)i] + deg[(size_t)i + 1];
    std::vector<int> fill(adj_ptr.begin(), adj_ptr.end() - 1), adj((size_t)adj_ptr[(size_t)n]);
    for (int f = 0; f < np; ++f) adj[(size_t)fill[(size_t)prior_node[f]]++] = (f << 2) | 2;
    for (int f = 0; f < nb; ++f) {
        adj[(size_t)fill[(size_t)bt_i[f]]++] = (f << 2) | 0;
        adj[(size_t)fill[(size_t)bt_j[f]]++] = (f << 2) | 1;
    }

    // ---- device state -----------------------------------------------------------------------------------------------------------------------
    DeviceArena A;
    cudaError_t ce = cudaSuccess;
    PgoView g{};
    g.n_nodes = n; g.n_prior = np; g.n_between = nb;
    g.prior_node = A.upload(prior_node, ce); g.prior_meas = A.upload(prior_meas, ce); g.prior_w = A.upload(prior_w, ce); g.prior_k = A.upload(prior_k, ce);
    g.bt_i = A.upload(bt_i, ce); g.bt_j = A.upload(bt_j, ce); g.bt_meas = A.upload(bt_meas, ce); g.bt_w = A.upload(bt_w, ce); g.bt_k = A.upload(bt_k, ce);
    g.we_prior = A.alloc<double>((size_t)np * 3, ce); g.we_bt = A.alloc<double>((size_t)nb * 3, ce);
    g.adj_ptr = A.upload(adj_ptr, ce); g.adj = A.upload(adj, ce);
    g.r_prior = A.alloc<double>((size_t)np * 3, ce); g.r_bt = A.alloc<double>((size_t)nb * 3, ce);
    g.J1 = A.alloc<double>((size_t)nb * 9, ce); g.B = A.alloc<double>((size_t)nb * 9, ce);
    g.D = A.alloc<double>((size_t)n * 9, ce); g.b = A.alloc<double>((size_t)n * 3, ce);
    SE2* X  = A.upload(nodes, ce);
    SE2* Xn = A.alloc<SE2>((size_t)n, ce);
    PcgBuffers w{};
    w.x = A.alloc<double>((size_t)n * 3, ce); w.r = A.alloc<double>((size_t)n * 3, ce); w.z = A.alloc<double>((size_t)n * 3, ce);
    w.p = A.alloc<double>((size_t)n * 3, ce); w.Ap = A.alloc<double>((size_t)n * 3, ce); w.Minv = A.alloc<double>((size_t)n * 9, ce);
    int sms = 0, per_sm = 0;
    if (ce == cudaSuccess) ce = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (ce == cudaSuccess) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pgo_pcg, 256, 0);
    int grid = std::max(1, std::min(sms * std::max(per_sm, 1), (n + 255) / 256));   // co-resident blocks only (cooperative launch)
    w.partial = A.alloc<double>((size_t)grid * 4, ce);
    w.out = A.alloc<double>(8, ce);
    const int err_blocks = 128;
    double* d_part = A.alloc<double>((size_t)err_blocks, ce);
    double* d_err  = A.alloc<double>(1, ce);
    Stream st;
    Event e0, e1;
    if (ce == cudaSuccess) ce = st.create();
    if (ce == cudaSuccess) ce = e0.create(cudaEventDefault);
    if (ce == cudaSuccess) ce = e1.create(cudaEventDefault);
    auto done = [&](int code, const std::string& what) {
        if (!what.empty()) err = what;
        return code;
    };
    if (ce != cudaSuccess) return done(LAMA_ERR_CUDA, std::string("pose graph: ") + cudaGetErrorString(ce));
    const int fb = (std::max(nb, np) + 127) / 128, nbk = (n + 127) / 128;
    auto graph_error = [&](const SE2* at, double* out) -> cudaError_t {   // 0.5 * errorSquaredNorm(values)
        k_pgo_linearize<<<fb, 128, 0, st>>>(g, at, 0);
        k_pgo_error_partial<<<err_blocks, 256, 0, st>>>(g, d_part);
        k_pgo_error_final<<<1, 32, 0, st>>>(d_part, err_blocks, d_err);
        cudaError_t e = cudaMemcpyAsync(out, d_err, 8, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        return e;
    };

    // ---- NonlinearOptimizer::optimize + LevenbergMarquardtOptimizer::iterate (host control in fp64, numbers from the device) ----------------
    const double lambda_max = 1e10, lambda_min = 1e-20, gain_thresh = 1e-3, dec_min = 1.0 / 3.0;   // LevenbergMarquardtOptimizer.h:21-36
    const uint32_t max_iterations = 100;                                                             // NonlinearOptimizer.h:54-58
    const double min_rel = 1e-5, min_abs = 1e-5;
    double lambda = 1e-5, inc = 2.0;
    const double cg_tol = 1e-10;    // relative residual of the damped normal equations
    int cg_max = 4 * n + 200;       // iteration cap of a solve; one that stops there above cg_tol gave a truncated step
    if (const char* cm = std::getenv("LAMA_PGO_CG_MAX")) {   // test hook: overrides the cap (a low one forces truncated solves)
        const int v = std::atoi(cm);
        if (v > 0) cg_max = v;
    }
    cudaEventRecord(e0, st);
    double last_err = 0;
    ce = graph_error(X, &last_err);                                                                  // NonlinearOptimizer.cpp:175
    if (ce != cudaSuccess) return done(LAMA_ERR_CUDA, std::string("pose graph: ") + cudaGetErrorString(ce));
    rep.initial_error = last_err;
    rep.status = 1;   // MAX_ITERATION unless decided otherwise
    while (rep.iterations < max_iterations) {
        k_pgo_linearize<<<fb, 128, 0, st>>>(g, X, 1);
        k_pgo_assemble<<<nbk, 128, 0, st>>>(g);
        bool accepted = false;
        double new_err = 0;
        while (lambda < lambda_max) {                                                                // LevenbergMarquardtOptimizer.cpp:121-151
            ++rep.lambda_tries;
            double lam = lambda, tol = cg_tol;
            int cap = cg_max;
            void* args[] = {&g, &w, &lam, &tol, &cap};
            ce = cudaLaunchCooperativeKernel((void*)k_pgo_pcg, dim3(grid), dim3(256), args, 0, st);
            if (ce != cudaSuccess) return done(LAMA_ERR_CUDA, std::string("pose graph: cooperative launch: ") + cudaGetErrorString(ce));
            k_pgo_retract<<<nbk, 128, 0, st>>>(n, X, w.x, Xn);
            double out[5];
            ce = cudaMemcpyAsync(out, w.out, sizeof(out), cudaMemcpyDeviceToHost, st);
            if (ce == cudaSuccess) ce = graph_error(Xn, &new_err);
            if (ce != cudaSuccess) return done(LAMA_ERR_CUDA, std::string("pose graph: ") + cudaGetErrorString(ce));
            rep.cg_iterations += (uint64_t)out[3];
            rep.accepted.push_back(0);
            // RANK_DEFICIENCY (SparseCholesky.cpp:26-31): a zero diagonal entry in a damped block, or a solve truncated at its cap above
            // the tolerance.  No step; lambda is raised and the next try goes on (LevenbergMarquardtOptimizer.cpp:139-144)
            const bool truncated = (int)out[3] >= cap && out[0] > tol * tol * out[1];
            const bool rank_deficient = out[4] != 0.0 || truncated;
            if (!rank_deficient && (!std::isfinite(out[0]) || !std::isfinite(out[2]))) { rep.status = 4; return done(LAMA_OK, ""); }   // INVALID
            const double nonlinear = last_err - new_err, linear = out[2];
            const double gain = nonlinear / linear;
            if (!rank_deficient && gain > gain_thresh) {                                             // :256-265
                rep.accepted.back() = 1;
                std::swap(X, Xn);
                lambda *= std::max(dec_min, 1.0 - std::pow(2.0 * gain - 1.0, 3.0));                  // decreaseLambda_ :342-348
                lambda = std::max(lambda_min, lambda);
                inc = 2.0;
                accepted = true;
                break;
            }
            lambda *= inc;                                                                           // increaseLambda_ :336-339
            inc *= 2.0;
        }
        ++rep.iterations;
        if (!accepted) { rep.status = 2; break; }                                                    // ERROR_INCREASE
        const double curr = new_err;
        if (curr - last_err > 1e-20) { rep.status = 2; break; }                                      // NonlinearOptimizer.cpp:213-216
        if ((last_err - curr) < min_abs || (last_err - curr) / last_err < min_rel) {                 // errorStopCondition_ :235-238
            last_err = curr;
            rep.status = 0;
            break;
        }
        last_err = curr;
    }
    rep.final_error = last_err;
    cudaEventRecord(e1, st);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    rep.device_ms = ms;
    if (rep.status == 0) {   // SimplePGO / GraphSlam2D take the result only on SUCCESS (simple_pgo.cpp:97-103, graph_slam2d.cpp:413-426)
        ce = cudaMemcpy(nodes.data(), X, (size_t)n * sizeof(SE2), cudaMemcpyDeviceToHost);
        if (ce != cudaSuccess) return done(LAMA_ERR_CUDA, std::string("pose graph: ") + cudaGetErrorString(ce));
    }
    return done(LAMA_OK, "");
}

int pgo_optimize(int device, std::vector<SE2>& nodes, const std::vector<PgoEdge>& edges, const std::vector<PgoFixed>& fixed, PgoReport& rep, std::string& err)
{
    rep = PgoReport();
    const int n = (int)nodes.size();
    if (n < 1) { err = "SimplePGO: no nodes"; return LAMA_ERR_ARG; }
    for (const PgoEdge& e : edges) {
        if (e.from < 0 || e.from >= n || e.to < 0 || e.to >= n) { err = "SimplePGO: edge index out of range"; return LAMA_ERR_ARG; }
        if (e.from == e.to) { err = "SimplePGO: an edge needs two distinct nodes (from == to)"; return LAMA_ERR_ARG; }
    }
    for (const PgoFixed& f : fixed)
        if (f.node < 0 || f.node >= n) { err = "SimplePGO: fixed node out of range"; return LAMA_ERR_ARG; }

    // ---- the factor graph of SimplePGO::optimize (simple_pgo.cpp:50-83) ---------------------------------------------------------------
    std::vector<PgoPrior> priors;
    if (fixed.empty()) {   // keep the first pose fixed: sigmas (1, 1, 1)
        priors.push_back(PgoPrior{0, nodes[0], PgoLoss{{1.0, 1.0, 1.0}, 0.0}});
    } else {               // sigmas (0.1, 0.1, 0.1)
        for (const PgoFixed& f : fixed) priors.push_back(PgoPrior{f.node, f.pose, PgoLoss{{0.1, 0.1, 0.1}, 0.0}});
    }
    const PgoLoss odom_loss{{0.5, 0.5, 0.1}, 0.0};   // odom_loss / loop_loss (:66, :76)
    std::vector<PgoBetween> betweens;
    for (int i = 0; i + 1 < n; ++i)   // odometry: node[i] - node[i + 1] = node[i]^-1 node[i + 1] (pose2d.cpp:81-84)
        betweens.push_back(PgoBetween{i, i + 1, se2_mul(se2_inv(nodes[(size_t)i]), nodes[(size_t)i + 1]), odom_loss});
    for (const PgoEdge& e : edges) betweens.push_back(PgoBetween{e.from, e.to, e.measured, odom_loss});
    return pgo_optimize_graph(device, nodes, priors, betweens, rep, err);
}

}  // namespace lama_b200
