// frontend.cpp -- host orchestration of PFSlam2D / Slam2D / Loc2D over the device Engine.
#include "frontend.h"
#include "checkpoint.h"
#include "rng_skip.h"

#include <cuda_runtime.h>

#include "shard_comm.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
#include <sstream>
#include <unordered_set>

namespace lama_b200 {

int cuda_device_count();  // engine.cu

SolverOptions make_solver(int strategy, uint32_t max_iter)
{
    SolverOptions so{};
    so.strategy       = strategy == 1 ? kStrategyLM : kStrategyGN;
    so.robust_kind    = kRobustCauchy;  // CauchyWeight(0.15): pf_slam2d.cpp:112,426 slam2d.cpp:107 loc2d.cpp:71
    so.robust_param   = 0.15;
    so.max_iterations = max_iter;
    so.eps1 = 1e-4;  // gauss_newton.cpp:40-41 / levenberg_marquardt.cpp:41-43
    so.eps2 = 1e-4;
    so.tau  = 1e-4;
    return so;
}

static EngineConfig engine_config(const DeviceOptions& dev, int particles, double resolution, double l2_max, double cx, double cy)
{
    EngineConfig c;
    c.device     = dev.device;
    c.particles  = particles;
    c.resolution = resolution;
    c.l2_max     = l2_max;
    c.dir_dim    = dev.dir_dim > 0 ? dev.dir_dim : 64;
    c.pool_slots = dev.pool_slots;
    c.max_beams  = dev.max_beams > 0 ? dev.max_beams : 2048;
    c.center_x   = cx;
    c.center_y   = cy;
    c.stream     = dev.stream;
    return c;
}

static double xy_norm(const SE2& s) { return std::sqrt(s.tx * s.tx + s.ty * s.ty); }

// =====================================================================================================
// PFSlam2D
// =====================================================================================================
PFSlam2D* PFSlam2D::create(const PFOptions& o, std::string& err)
{
    if (o.particles < 1) { err = "PFSlam2D: Options::particles must be set (>= 1)"; return nullptr; }
    if (o.patch_size != 32) { err = "PFSlam2D: only patch_size 32 is supported on the device"; return nullptr; }
    if (o.shard_count < 1 || o.shard_rank >= o.shard_count || o.particles % o.shard_count != 0) {
        err = "PFSlam2D: particles must divide evenly over shard_count";
        return nullptr;
    }
    if (o.shard_count > 1 && o.seed == 0) {
        // seed 0 means "take one from random_device" (pf_slam2d.cpp:131-132): every rank would draw its own, the ranks' odometry
        // noise and resampling indices would differ and the map migration would pair up the wrong particles
        err = "PFSlam2D: sharded operation needs an explicit (non-zero) seed shared by all ranks";
        return nullptr;
    }
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    PFSlam2D* p = new PFSlam2D();
    p->opt_ = o;
    p->P_   = o.particles;
    const int per = (int)(o.particles / o.shard_count);
    p->lo_ = (int)o.shard_rank * per;
    p->hi_ = p->lo_ + per;
    if (p->opt_.seed == 0) p->opt_.seed = std::random_device{}();  // pf_slam2d.cpp:131-132
    p->gen_.seed(p->opt_.seed);                                    // random::setSeed, pf_slam2d.cpp:134
    p->pose_.assign(p->P_, SE2{1, 0, 0, 0});
    p->weight_.assign(p->P_, 0.0);
    p->nweight_.assign(p->P_, 0.0);
    p->wsum_.assign(p->P_, 0.0);
    p->node_of_.assign(p->P_, -1);
    return p;
}
PFSlam2D::~PFSlam2D()
{
    if (comm_) {
        shard_comm_destroy(comm_);
        cudaFree(d_send_);
        cudaFree(d_recv_);
        cudaFree(d_tab_);
        cudaFreeHost(h_recv_);
        cudaFreeHost(h_tab_);
    }
}

double PFSlam2D::rng_normal(double sigma)  // random::normal, src/random.cpp:69-73
{
    std::normal_distribution<double> d(0.0, sigma);
    return d(gen_);
}
double PFSlam2D::rng_uniform()  // random::uniform, src/random.cpp:51-55
{
    std::uniform_real_distribution<double> d(0.0, 1.0);
    return d(gen_);
}

void PFSlam2D::draw_from_motion(const SE2& delta, SE2& p)
{
    const double dx = delta.tx, dy = delta.ty, dr = se2_rotation(delta);
    double sigma, x, y, yaw;
    const double sxy = 0.3 * opt_.stt;
    sigma = opt_.stt * std::fabs(dx) + opt_.str * std::fabs(dr) + sxy * std::fabs(dy);
    x     = dx + rng_normal(sigma);
    sigma = opt_.stt * std::fabs(dy) + opt_.str * std::fabs(dr) + sxy * std::fabs(dx);
    y     = dy + rng_normal(sigma);
    sigma = opt_.srr * std::fabs(dr) + opt_.srt * xy_norm(delta);
    yaw   = dr + rng_normal(sigma);
    yaw   = std::fmod(yaw, 2 * M_PI);
    if (yaw > M_PI) yaw -= 2 * M_PI;
    p = se2_mul(p, se2_from_xyr(x, y, yaw));
}

int PFSlam2D::first_scan(const double odom_xyr[3])
{
    // pf_slam2d.cpp:185-228
    odom_ = se2_from_xyr(odom_xyr[0], odom_xyr[1], odom_xyr[2]);
    for (uint32_t i = 0; i < P_; ++i) {
        pose_[i]    = prior_;
        weight_[i]  = 0.0;
        wsum_[i]    = 0.0;
        nodes_.push_back(Node{prior_, -1});
        node_of_[i] = (int)nodes_.size() - 1;
    }
    const int nl = hi_ - lo_;
    HostMapStats st{};
    int rc = eng_->update_maps(&prior_, 0, 1, &st);  // particle 0's maps are built from the scan ...
    if (rc != LAMA_OK) return engine_fail(rc);
    rc = eng_->share_from(0, 1, nl - 1);              // ... and COW-shared with all the others (:208-216)
    if (rc != LAMA_OK) return engine_fail(rc);
    last_.ray_cells = st.ray_cells;
    last_.dm_pops   = st.dm_pops;
    has_first_      = true;
    return LAMA_OK;
}

bool PFSlam2D::predict_and_gate(const double odom_xyr[3])
{
    const SE2 odometry = se2_from_xyr(odom_xyr[0], odom_xyr[1], odom_xyr[2]);
    const SE2 odelta   = se2_mul(se2_inv(odom_), odometry);  // Pose2D::operator-, pose2d.cpp:81-84
    odom_ = odometry;
    acc_trans_ += xy_norm(odelta);
    acc_rot_ += std::fabs(se2_rotation(odelta));
    const bool moved = !(acc_trans_ <= opt_.trans_thresh && acc_rot_ <= opt_.rot_thresh);   // the gate does not depend on the samples
    // Every rank draws the noise of ALL particles, so that the random streams stay identical.  On a scan that will be matched the predicted poses of
    // the other ranks' particles are never read (absorb_results replaces them with the gathered match results): for those only the generator is
    // advanced (rng_skip.h) -- 1.8 k of 2 k particles at 8 ranks.  A gated scan keeps the predictions, so there every pose is computed.
    for (uint32_t i = 0; i < P_; ++i) {
        if (moved && ((int)i < lo_ || (int)i >= hi_)) {
            rng_skip_normal(gen_);
            rng_skip_normal(gen_);
            rng_skip_normal(gen_);
        } else {
            draw_from_motion(odelta, pose_[i]);
        }
    }
    if (!moved) return false;
    acc_trans_ = 0;
    acc_rot_   = 0;
    return true;
}

int PFSlam2D::match_local(double* local_out)
{
    const int nl = hi_ - lo_;
    std::vector<HostMatchResult> res((size_t)nl);
    // PFSlam2D::scanMatch always uses GaussNewton + CauchyWeight(0.15), pf_slam2d.cpp:423-427
    SolverOptions so = make_solver(0, opt_.max_iter);
    int rc = eng_->match(&pose_[lo_], nl, 0, false, so, opt_.meas_sigma, 0, res.data());
    if (rc != LAMA_OK) return engine_fail(rc);
    for (int k = 0; k < nl; ++k) {
        local_out[5 * k + 0] = res[k].state.c;
        local_out[5 * k + 1] = res[k].state.s;
        local_out[5 * k + 2] = res[k].state.tx;
        local_out[5 * k + 3] = res[k].state.ty;
        local_out[5 * k + 4] = res[k].sums[11];  // calculateLikelihood, pf_slam2d.cpp:393-414
        last_.evals += res[k].evals_ref + 1;     // + the likelihood pass
        last_.gn_iters += res[k].iterations;
    }
    return LAMA_OK;
}

void PFSlam2D::absorb_results(const double* all)
{
    ++scans_seen_;
    for (uint32_t i = 0; i < P_; ++i) {
        pose_[i] = SE2{all[5 * i], all[5 * i + 1], all[5 * i + 2], all[5 * i + 3]};
        nodes_.push_back(Node{pose_[i], node_of_[i]});  // particle->poses.push_back(pose)
        node_of_[i] = (int)nodes_.size() - 1;
        const double l = all[5 * i + 4];
        wsum_[i] += l;
        weight_[i] += l;
    }
}

void PFSlam2D::normalize()
{
    const double gain = 1.0 / (opt_.meas_sigma_gain * opt_.particles);
    double max_l = weight_[0];
    for (uint32_t i = 1; i < P_; ++i)
        if (max_l < weight_[i]) max_l = weight_[i];
    double sum = 0;
    for (uint32_t i = 0; i < P_; ++i) {
        nweight_[i] = std::exp(gain * (weight_[i] - max_l));
        sum += nweight_[i];
    }
    neff_ = 0;
    for (uint32_t i = 0; i < P_; ++i) {
        nweight_[i] /= sum;
        neff_ += nweight_[i] * nweight_[i];
    }
    neff_ = 1.0 / neff_;
}

bool PFSlam2D::compute_resample(std::vector<int32_t>& idx)
{
    if (!(neff_ < (opt_.particles * 0.5))) return false;  // pf_slam2d.cpp:279
    idx.assign(P_, 0);
    const double interval = 1.0 / (double)P_;
    double target = interval * rng_uniform();
    double cw = 0.0;
    uint32_t n = 0;
    for (size_t i = 0; i < P_; ++i) {
        cw += nweight_[i];
        while (cw > target) {
            if (n < P_) idx[n] = (int32_t)i;  // the reference writes sample_idx[n++] unguarded (:550-553)
            ++n;
            target += interval;
        }
    }
    return true;
}

void PFSlam2D::note_resample(const std::vector<int32_t>& idx)
{
    auto mix = [this](uint64_t v) {
        for (int k = 0; k < 8; ++k) { resample_hash_ ^= (v >> (8 * k)) & 0xFFu; resample_hash_ *= 1099511628211ull; }
    };
    ++resample_count_;
    mix(scans_seen_);
    for (int32_t i : idx) mix((uint64_t)(uint32_t)i);
}

void PFSlam2D::apply_resample_host(const std::vector<int32_t>& idx)
{
    note_resample(idx);
    std::vector<SE2> np(P_);
    std::vector<double> nw(P_), nn(P_), ns(P_);
    std::vector<int> nnode(P_);
    for (uint32_t i = 0; i < P_; ++i) {
        const int a = idx[i];
        np[i]    = pose_[a];
        nw[i]    = 0.0;
        nn[i]    = nweight_[a];
        ns[i]    = wsum_[a];
        nnode[i] = node_of_[a];
    }
    pose_.swap(np);
    weight_.swap(nw);
    nweight_.swap(nn);
    wsum_.swap(ns);
    node_of_.swap(nnode);
}

int PFSlam2D::settle_counters()
{
    if (!counters_pending_) return LAMA_OK;
    counters_pending_ = false;
    int rc = eng_->settle(nullptr);
    for (const HostMapStats& st : eng_->last_map_stats()) {
        last_.ray_cells += st.ray_cells;
        last_.dm_pops += st.dm_pops;
    }
    finish_counters();
    return rc == LAMA_OK ? rc : engine_fail(rc);
}

void PFSlam2D::finish_counters()
{
    uint64_t c[4];
    eng_->store_counters(c);
    last_.detached = c[1] - detached_seen_;
    detached_seen_ = c[1];
    total_.add(last_);
}

// The whole scan enqueued at once (Engine::step_async): odometry sampling on the host, then match -> ray cast -> brushfire
// back to back on the device.  The map update runs on the matched poses BEFORE the resampling decision; a resampling of
// this scan then shares the UPDATED maps, which is the reference's resample-then-update with the two steps commuted
// (every copy of an ancestor would apply the same scan at the same pose).  The host only waits for the match results.
// Front half of a pipelined step for the local particles [lo_, hi_): enqueue match + map update, wait for the match results only,
// then book the previous scan's map statistics (its map update precedes this scan's match in the stream, so it has completed).
// `moved` false = motion gate (pf_slam2d.cpp:215-222): nothing else happens for this scan.
int PFSlam2D::pipelined_begin(const double* pts, int n, const double* origin, const double* quat, bool moved, bool* did_update, double* local_out)
{
    pending_maps_ = false;
    if (!moved) {
        int rcs = settle_counters();
        last_ = Counters();
        last_idx_.clear();
        staged_index_ = -1;
        return rcs;
    }
    *did_update = true;
    Counters prev = last_;
    const bool prev_pending = counters_pending_;
    counters_pending_ = false;
    last_ = Counters();
    last_idx_.clear();
    const int staged = staged_index_;
    staged_index_ = -1;
    int rc = LAMA_OK;
    if (staged >= 0) {
        rc = eng_->select_staged(staged, origin, quat, opt_.truncated_ray, opt_.truncated_range);
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    const int nl = hi_ - lo_;
    std::vector<HostMatchResult> res((size_t)nl);
    rc = eng_->step_async(staged >= 0 ? nullptr : pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range, &pose_[lo_], nl,
                          make_solver(0, opt_.max_iter), opt_.meas_sigma, res.data());   // GaussNewton + CauchyWeight(0.15), pf_slam2d.cpp:423-427
    if (prev_pending) {
        collect_map_stats(prev);
        total_.add(prev);
    }
    if (rc != LAMA_OK) return engine_fail(rc);
    for (int k = 0; k < nl; ++k) {
        local_out[5 * k + 0] = res[k].state.c;
        local_out[5 * k + 1] = res[k].state.s;
        local_out[5 * k + 2] = res[k].state.tx;
        local_out[5 * k + 3] = res[k].state.ty;
        local_out[5 * k + 4] = res[k].sums[11];  // calculateLikelihood, pf_slam2d.cpp:393-414
        last_.evals += res[k].evals_ref + 1;     // + the likelihood pass
        last_.gn_iters += res[k].iterations;
    }
    return LAMA_OK;
}

// The whole scan enqueued at once (Engine::step_async): odometry sampling on the host, then match -> ray cast -> brushfire
// back to back on the device.  The map update runs on the matched poses BEFORE the resampling decision; a resampling of
// this scan then shares the UPDATED maps, which is the reference's resample-then-update with the two steps commuted
// (every copy of an ancestor would apply the same scan at the same pose).  The host only waits for the match results.
int PFSlam2D::update_pipelined(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], bool* did_update)
{
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = clk::now();
    const bool moved = predict_and_gate(odom_xyr);
    const auto t1 = clk::now();
    t_sample_ += ms(t0, t1);
    std::vector<double> all((size_t)P_ * 5);
    int rc = pipelined_begin(pts, n, origin, quat, moved, did_update, all.data());
    const auto t2 = clk::now();
    t_solve_ += ms(t1, t2);
    if (rc != LAMA_OK || !moved) return rc;
    absorb_results(all.data());
    normalize();
    const auto t3 = clk::now();
    t_norm_ += ms(t2, t3);
    std::vector<int32_t> v;
    counters_pending_ = true;
    struct Stop { clk::time_point t; double& acc; ~Stop() { acc += std::chrono::duration<double, std::milli>(clk::now() - t).count(); } } stop{t3, t_resample_};
    if (compute_resample(v)) {
        apply_resample_host(v);
        last_idx_ = v;
        last_.resampled = 1;
        std::vector<int32_t> src(v.begin(), v.end());
        rc = eng_->resample(src.data());   // after this scan's map update in stream order: the offspring share the updated maps
        if (rc != LAMA_OK) return engine_fail(rc);
        // resample() waited for the map update and collected it
        collect_map_stats(last_);
        total_.add(last_);
        counters_pending_ = false;
    }
    return LAMA_OK;
}

void PFSlam2D::collect_map_stats(Counters& c)
{
    for (const HostMapStats& st : eng_->last_map_stats()) {
        c.ray_cells += st.ray_cells;
        c.dm_pops += st.dm_pops;
    }
    const uint64_t* sc = eng_->settled_store_counters();
    c.detached     = sc[1] - detached_seen_;
    detached_seen_ = sc[1];
}

// ---- sharded update over NCCL ---------------------------------------------------------------------------------------------------
constexpr int kShardF = 7;   // kernels.cuh kShardFields: state (4), likelihood, reference evaluations, iterations

int PFSlam2D::shard_connect(const uint8_t id[128])
{
    if (opt_.shard_count < 2) return fail("shard_connect: the handle was created with shard_count 1", LAMA_ERR_STATE);
    if (comm_) return fail("shard_connect: already connected", LAMA_ERR_STATE);
    std::string e;
    comm_ = shard_comm_create(id, (int)opt_.shard_rank, (int)opt_.shard_count, opt_.dev.device, e);
    if (!comm_) return fail(e, LAMA_ERR_CUDA);
    const size_t per = (size_t)(hi_ - lo_), payload = per * kShardF + 1;
    bool ok = cudaMalloc((void**)&d_send_, payload * 8) == cudaSuccess && cudaMalloc((void**)&d_recv_, payload * 8 * opt_.shard_count) == cudaSuccess &&
              cudaMallocHost((void**)&h_recv_, payload * 8 * opt_.shard_count) == cudaSuccess && cudaMalloc((void**)&d_tab_, (size_t)P_ * 3 * 8 * 2) == cudaSuccess &&
              cudaMallocHost((void**)&h_tab_, (size_t)P_ * 3 * 8 * 2) == cudaSuccess;
    if (!ok) return fail("shard_connect: out of memory", LAMA_ERR_CUDA);
    return LAMA_OK;
}

// One sharded step, the same on every rank (src/pf_slam2d.cpp:178-312 with the two fan-outs :254-266,:292-302 running on this rank's
// particles only).  Every rank draws the odometry noise of ALL particles (identical generators), enqueues match + map update of its
// shard, and all-gathers {state, likelihood, counts} of the local particles plus a digest of its previous resampling decision -- one
// collective per scan.  Normalise / resample then run on identical bytes with identical generator states on every rank.
int PFSlam2D::update_sharded(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], bool* did_update)
{
    *did_update = false;
    if (!has_first_) {   // first scan: every rank builds its own copy from the prior, nothing to exchange (pf_slam2d.cpp:185-228)
        std::vector<double> dummy((size_t)(hi_ - lo_) * 5);
        return shard_begin(pts, n, origin, quat, odom_xyr, 0.0, did_update, dummy.data());
    }
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = clk::now();
    const bool moved = predict_and_gate(odom_xyr);
    const auto t1 = clk::now();
    t_sample_ += ms(t0, t1);
    if (!moved) {
        int rcs = settle_counters();
        last_ = Counters();
        last_idx_.clear();
        staged_index_ = -1;
        return rcs;
    }
    *did_update = true;
    Counters prev = last_;
    const bool prev_pending = counters_pending_;
    counters_pending_ = false;
    last_ = Counters();
    last_idx_.clear();
    const int staged = staged_index_;
    staged_index_ = -1;
    int rc = LAMA_OK;
    if (staged >= 0) {
        rc = eng_->select_staged(staged, origin, quat, opt_.truncated_ray, opt_.truncated_range);
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    const int nl = hi_ - lo_, G = (int)opt_.shard_count;
    rc = eng_->step_enqueue(staged >= 0 ? nullptr : pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range, &pose_[lo_], nl, make_solver(0, opt_.max_iter),
                            opt_.meas_sigma);
    if (rc != LAMA_OK) return engine_fail(rc);
    const size_t payload = (size_t)nl * kShardF + 1;
    rc = eng_->pack_results(nl, digest_, d_send_, shard_stream(comm_));   // waits for the match on the communicator's stream
    if (rc != LAMA_OK) return engine_fail(rc);
    if (shard_allgather(comm_, d_send_, d_recv_, payload * 8) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    if (cudaMemcpyAsync(h_recv_, d_recv_, payload * 8 * G, cudaMemcpyDeviceToHost, (cudaStream_t)shard_stream(comm_)) != cudaSuccess)
        return fail("update_sharded: copy of the gathered results failed", LAMA_ERR_CUDA);
    if (shard_sync(comm_) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    ++shard_collectives_;
    rc = eng_->collect_previous();   // the previous scan's map update precedes this scan's match in the engine's stream
    if (prev_pending) {
        collect_map_stats(prev);
        total_.add(prev);
    }
    if (rc != LAMA_OK) return engine_fail(rc);
    const auto t2 = clk::now();
    t_solve_ += ms(t1, t2);
    std::vector<double> all((size_t)P_ * 5);
    for (int r = 0; r < G; ++r) {
        const double* src = h_recv_ + (size_t)r * payload;
        if (src[(size_t)nl * kShardF] != h_recv_[(size_t)nl * kShardF]) return fail("the resampling decision diverged between ranks", LAMA_ERR_STATE);
        for (int k = 0; k < nl; ++k) {
            const double* f = src + (size_t)k * kShardF;
            double* dst = &all[((size_t)r * nl + k) * 5];
            dst[0] = f[0]; dst[1] = f[1]; dst[2] = f[2]; dst[3] = f[3]; dst[4] = f[4];
            last_.evals += (uint64_t)f[5] + 1;   // + the likelihood pass
            last_.gn_iters += (uint64_t)f[6];
        }
    }
    absorb_results(all.data());
    normalize();
    const auto t3 = clk::now();
    t_norm_ += ms(t2, t3);
    std::vector<int32_t> v;
    const bool res = compute_resample(v);
    digest_ = 0.0;
    if (res) {
        uint64_t acc = 1;
        for (uint32_t i = 0; i < P_; ++i) acc = (acc + (uint64_t)(uint32_t)v[i] * (uint64_t)(i + 1)) % 9007199254740881ull;
        digest_ = (double)acc;
        rc = migrate_and_apply(v);
        if (rc != LAMA_OK) return rc;
        last_.resampled = 1;
    }
    t_resample_ += ms(t3, clk::now());
    counters_pending_ = !res;   // this scan's map update is still running; after a resampling it has been waited for and booked already
    return LAMA_OK;
}

// Resampling across ranks: the offspring of a remote ancestor need its (already updated) maps.  Who needs what follows from the
// indices alone, which every rank holds; only the blob sizes are exchanged first (one small all-gather), then all blobs move in one
// grouped NCCL send / recv between device arenas.
int PFSlam2D::migrate_and_apply(const std::vector<int32_t>& idx)
{
    const int G = (int)opt_.shard_count, per = hi_ - lo_, me = (int)opt_.shard_rank;
    // need[r]: sorted unique remote ancestors of rank r's new particles; serve: (destination, ancestor) pairs this rank sends
    std::vector<std::vector<int>> need((size_t)G);
    for (int r = 0; r < G; ++r) {
        std::vector<int> a(idx.begin() + (size_t)r * per, idx.begin() + (size_t)(r + 1) * per);
        std::sort(a.begin(), a.end());
        a.erase(std::unique(a.begin(), a.end()), a.end());
        for (int g : a)
            if (g / per != r) need[(size_t)r].push_back(g);
    }
    std::vector<std::pair<int, int>> serve;
    for (int r = 0; r < G; ++r)
        for (int g : need[(size_t)r])
            if (g / per == me) serve.push_back({r, g});
    // pack every local particle somebody needs (once), after this scan's map update has finished (pack_device settles)
    std::vector<Engine::DeviceBlob> blob((size_t)per);
    std::vector<int64_t> mine((size_t)per * 3, 0);
    for (const auto& sv : serve) {
        const int k = sv.second - lo_;
        if (blob[(size_t)k].dptr) continue;
        int rc = eng_->pack_device(k, &blob[(size_t)k]);
        if (rc != LAMA_OK) return engine_fail(rc);
        mine[(size_t)k * 3] = (int64_t)blob[(size_t)k].bytes; mine[(size_t)k * 3 + 1] = blob[(size_t)k].n_occ; mine[(size_t)k * 3 + 2] = blob[(size_t)k].n_dm;
    }
    cudaStream_t cs = (cudaStream_t)shard_stream(comm_);
    // the gather kernels of the packs run on the engine's stream; everything the communicator's stream does from here on (the sends) comes after them
    if (eng_->wait_for_stream(cs) != LAMA_OK) return engine_fail(LAMA_ERR_CUDA);
    std::memcpy(h_tab_, mine.data(), mine.size() * 8);
    int64_t* d_all = d_tab_ + (size_t)P_ * 3;
    int64_t* h_all = h_tab_ + (size_t)P_ * 3;
    if (cudaMemcpyAsync(d_tab_, h_tab_, mine.size() * 8, cudaMemcpyHostToDevice, cs) != cudaSuccess) return fail("migrate: size table upload failed", LAMA_ERR_CUDA);
    if (shard_allgather(comm_, d_tab_, d_all, mine.size() * 8) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    if (cudaMemcpyAsync(h_all, d_all, (size_t)P_ * 3 * 8, cudaMemcpyDeviceToHost, cs) != cudaSuccess) return fail("migrate: size table download failed", LAMA_ERR_CUDA);
    if (shard_sync(comm_) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    ++shard_collectives_;
    std::vector<ShardXfer> sends, recvs;
    for (const auto& sv : serve) {
        const Engine::DeviceBlob& b = blob[(size_t)(sv.second - lo_)];
        if (b.bytes) sends.push_back({sv.first, b.dptr, b.bytes});
    }
    std::vector<Engine::DeviceBlob> in(need[(size_t)me].size());
    for (size_t k = 0; k < in.size(); ++k) {
        const int g = need[(size_t)me][k];
        in[k].bytes = (size_t)h_all[(size_t)g * 3]; in[k].n_occ = (uint32_t)h_all[(size_t)g * 3 + 1]; in[k].n_dm = (uint32_t)h_all[(size_t)g * 3 + 2];
        int rc = eng_->migration_alloc(in[k].bytes, &in[k].dptr);
        if (rc != LAMA_OK) return engine_fail(rc);
        if (in[k].bytes) recvs.push_back({g / per, in[k].dptr, in[k].bytes});
        shard_migrated_bytes_ += in[k].bytes;
    }
    if (shard_exchange(comm_, sends, recvs) != 0 || shard_sync(comm_) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    if (!sends.empty() || !recvs.empty()) ++shard_collectives_;
    std::vector<int32_t> local_src((size_t)per);
    for (size_t k = 0; k < in.size(); ++k) {
        int rc = eng_->unpack_device(per + (int)k, in[k], k + 1 == in.size());   // staging slots behind the local particles; one status check for all
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    for (int k = 0; k < per; ++k) {
        const int g = idx[(size_t)lo_ + k];
        if (g / per == me) local_src[(size_t)k] = g - lo_;
        else local_src[(size_t)k] = per + (int)(std::lower_bound(need[(size_t)me].begin(), need[(size_t)me].end(), g) - need[(size_t)me].begin());
    }
    eng_->migration_reset();
    pending_maps_ = true;   // shard_apply's precondition
    int rc = shard_apply(idx.data(), local_src.data());
    pending_maps_ = false;
    if (rc != LAMA_OK) return rc;
    // resample() waited for the map update and collected it
    collect_map_stats(last_);
    total_.add(last_);
    return LAMA_OK;
}

int PFSlam2D::memory_usage(uint64_t out[3])
{
    out[0] = out[1] = out[2] = 0;
    if (!has_first_ || !eng_) return LAMA_OK;
    const int local = eng_->config().particles;
    std::vector<uint64_t> occ((size_t)local), dm((size_t)local);
    // sizeof(frequency) = 4 (frequency_occupancy_map.h), sizeof(distance_t) = 10 (dynamic_distance_map.h: three int16, uint16, two bool)
    if (eng_->memory_usage(0 /* occupancy */, 4u, occ.data()) != 0 || eng_->memory_usage(1 /* distance */, 10u, dm.data()) != 0) return engine_fail(LAMA_ERR_CUDA);
    for (int i = 0; i < local; ++i) out[0] += occ[(size_t)i] + dm[(size_t)i];
    out[1] = occ[0] * (uint64_t)local;
    out[2] = dm[0] * (uint64_t)local;
    return LAMA_OK;
}

int PFSlam2D::update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update)
{
    if (!has_first_) timestamps_.push_back(stamp);
    if (opt_.shard_count != 1) {
        if (!comm_) return fail("PFSlam2D::update on a sharded handle: connect the ranks first (lama_pf_shard_connect) or use the split-phase shard_* calls", LAMA_ERR_STATE);
        bool did = false;
        int rc = update_sharded(pts, n, origin, quat, odom_xyr, &did);
        if (did_update) *did_update = did;
        return rc;
    }
    if (has_first_ && eng_ && opt_.dev.timing == 0) {
        bool did = false;
        int rc = update_pipelined(pts, n, origin, quat, odom_xyr, &did);
        if (did_update) *did_update = did;
        return rc;
    }
    std::vector<double> local((size_t)P_ * 5);
    bool did = false;
    int rc = shard_begin(pts, n, origin, quat, odom_xyr, stamp, &did, local.data());
    if (did_update) *did_update = did;
    if (rc != LAMA_OK || !did || !pending_maps_) return rc;
    bool resampled = false;
    std::vector<int32_t> idx(P_);
    rc = shard_finish(local.data(), &resampled, idx.data());
    if (rc != LAMA_OK) return rc;
    if (resampled) {
        rc = shard_apply(idx.data(), idx.data());
        if (rc != LAMA_OK) return rc;
    }
    return shard_map_update();
}

int PFSlam2D::shard_begin(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double, bool* did_update,
                          double* local_out)
{
    *did_update   = false;
    pending_maps_ = false;
    // Host-only work first: the odometry sampling of this scan (global mt19937, all particles, in order) does not
    // depend on the previous scan's map update, which may still be running on the device.
    bool moved = false;
    if (has_first_) moved = predict_and_gate(odom_xyr);
    if (has_first_ && eng_ && opt_.shard_count > 1 && opt_.dev.timing == 0) {
        // Sharded ranks: the map update of the local particles is enqueued right behind their match and runs while the ranks
        // exchange results and decide about resampling; a resampling of this scan then moves / shares the UPDATED maps.
        maps_enqueued_ = false;
        int rcp = pipelined_begin(pts, n, origin, quat, moved, did_update, local_out);
        if (rcp != LAMA_OK || !moved) return rcp;
        maps_enqueued_ = true;
        pending_maps_  = true;
        return LAMA_OK;
    }
    if (eng_) {
        int rcs = settle_counters();   // now collect the previous scan's asynchronous map update (and its errors)
        if (rcs != LAMA_OK) return rcs;
    }
    last_ = Counters();
    last_idx_.clear();
    int rc = ensure_engine(staged_index_ >= 0 ? staged_beams_ : n);
    if (rc != LAMA_OK) return rc;
    if (staged_index_ >= 0) rc = eng_->select_staged(staged_index_, origin, quat, opt_.truncated_ray, opt_.truncated_range);
    else rc = eng_->set_scan(pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range);
    staged_index_ = -1;
    if (rc != LAMA_OK) return engine_fail(rc);
    if (!has_first_) {
        rc = first_scan(odom_xyr);
        if (rc != LAMA_OK) return rc;
        *did_update = true;
        finish_counters();
        return LAMA_OK;
    }
    if (!moved) return LAMA_OK;
    *did_update = true;
    maps_enqueued_ = false;
    rc = match_local(local_out);
    if (rc != LAMA_OK) return rc;
    pending_maps_ = true;
    return LAMA_OK;
}

int PFSlam2D::ensure_engine(int n)
{
    if (eng_) return LAMA_OK;
    // device state is created on the first scan, centred on the prior
    std::string e;
    EngineConfig cfg = engine_config(opt_.dev, 2 * (hi_ - lo_), opt_.resolution, opt_.l2_max, prior_.tx, prior_.ty);
    if (opt_.shard_count == 1) cfg.particles = hi_ - lo_;  // no staging slots needed without migration
    cfg.max_beams = std::max(cfg.max_beams, n);
    Engine* en = Engine::create(cfg, e);
    if (!en) return fail(e, LAMA_ERR_CUDA);
    eng_.reset(en);
    eng_->enable_timing(opt_.dev.timing != 0);
    if (!staged_host_.empty()) {
        int rc = eng_->stage_scans(staged_host_.data(), staged_scans_, staged_beams_);
        staged_host_.clear();
        staged_host_.shrink_to_fit();
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    return LAMA_OK;
}

int PFSlam2D::stage_scans(const double* pts, int n_scans, int n)
{
    if (!pts || n_scans < 1 || n < 1) return fail("stage_scans: bad arguments", LAMA_ERR_ARG);
    staged_scans_ = n_scans;
    staged_beams_ = n;
    if (eng_) {
        int rc = eng_->stage_scans(pts, n_scans, n);
        return rc == LAMA_OK ? rc : engine_fail(rc);
    }
    staged_host_.assign(pts, pts + (size_t)n_scans * n * 3);
    return LAMA_OK;
}

int PFSlam2D::update_staged(int index, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update)
{
    if (index < 0 || index >= staged_scans_) return fail("update_staged: no such staged scan", LAMA_ERR_ARG);
    staged_index_ = index;
    return update(nullptr, staged_beams_, origin, quat, odom_xyr, stamp, did_update);
}

int PFSlam2D::shard_finish(const double* all_results, bool* resampled, int32_t* idx)
{
    if (!pending_maps_) return fail("shard_finish without a pending update", LAMA_ERR_STATE);
    absorb_results(all_results);
    normalize();
    std::vector<int32_t> v;
    *resampled = compute_resample(v);
    if (*resampled) std::copy(v.begin(), v.end(), idx);
    return LAMA_OK;
}

int PFSlam2D::shard_apply(const int32_t* idx, const int32_t* local_src)
{
    if (!pending_maps_) return fail("shard_apply without a pending update", LAMA_ERR_STATE);
    std::vector<int32_t> v(idx, idx + P_);
    apply_resample_host(v);
    last_idx_ = v;
    last_.resampled = 1;
    // device side: new local particle k takes the maps of engine slot src[k]
    const int nl = hi_ - lo_;
    std::vector<int32_t> src((size_t)eng_->config().particles, 0);
    for (int k = 0; k < nl; ++k) src[k] = (opt_.shard_count == 1) ? idx[lo_ + k] : local_src[k];
    for (int k = nl; k < eng_->config().particles; ++k) src[k] = -1;
    int rc = eng_->resample(src.data());
    if (rc != LAMA_OK) return engine_fail(rc);
    return LAMA_OK;
}

int PFSlam2D::shard_map_update()
{
    if (!pending_maps_) return fail("shard_map_update without a pending update", LAMA_ERR_STATE);
    pending_maps_ = false;
    const int nl = hi_ - lo_;
    if (maps_enqueued_) {   // already running since shard_begin
        maps_enqueued_    = false;
        counters_pending_ = true;
        return LAMA_OK;
    }
    // asynchronous: the kernels of this scan overlap with the caller's work until the next call into this handle
    int rc = eng_->update_maps_async(&pose_[lo_], 0, nl);
    if (rc != LAMA_OK) return engine_fail(rc);
    counters_pending_ = true;
    return LAMA_OK;
}

size_t PFSlam2D::best_particle() const
{
    size_t best = 0;
    double ws   = wsum_[0];
    for (uint32_t i = 1; i < P_; ++i)
        if (ws < wsum_[i]) {
            ws   = wsum_[i];
            best = i;
        }
    return best;
}

std::vector<SE2> PFSlam2D::trajectory(int particle) const
{
    std::vector<SE2> out;
    for (int n = node_of_[particle]; n >= 0; n = nodes_[n].parent) out.push_back(nodes_[n].pose);
    std::reverse(out.begin(), out.end());
    return out;
}

// =====================================================================================================
// GraphSlam2D loop-closure front end (src/graph_slam2d.cpp:283-392)
// =====================================================================================================
std::vector<int> find_loop_closure_candidates(const double* key_xy, int n_keys, int ignore_n, const double query[2], double radius, int max_candidates)
{
    std::vector<std::pair<double, int>> hits;
    const int n = n_keys - ignore_n;   // KeyPosesNanoFlannAdaptor::kdtree_get_point_count (:73)
    for (int i = 0; i < n; ++i) {
        const double dx = key_xy[2 * i] - query[0], dy = key_xy[2 * i + 1] - query[1];
        const double d2 = dx * dx + dy * dy;   // L2_Simple_Adaptor: squared distance; radiusSearch keeps d2 < radius^2 (:296)
        if (d2 < radius * radius) hits.push_back({d2, i});
    }
    std::sort(hits.begin(), hits.end(), [](const std::pair<double, int>& a, const std::pair<double, int>& b) { return a.first < b.first; });   // IndexDist_Sorter
    if ((int)hits.size() > max_candidates) hits.resize((size_t)max_candidates);                                                               // :298-301
    std::vector<int> out;
    for (const auto& h : hits) out.push_back(h.second);
    return out;
}

static SolverOptions huber_solver(uint32_t max_iter)
{
    SolverOptions so = make_solver(0, max_iter);   // GaussNewton (:324)
    so.robust_kind  = kRobustHuber;                // HuberWeight(0.15) (:325)
    so.robust_param = 0.15;
    return so;
}

int correlate_candidate_scan(Engine* e, int particle, const double* pts, int n, const double* origin, const double* quat, const SE2& ref_pose, const SE2& cand_pose,
                             SE2* between, double* rmse)
{
    int rc = e->set_scan(pts, n, origin, quat, 0, 0);
    if (rc != LAMA_OK) return rc;
    // the two starts (:328-329): the candidate's own pose, and the reference position with the candidate's heading
    SE2 st[2] = {cand_pose, se2_from_xyr(ref_pose.tx, ref_pose.ty, se2_rotation(cand_pose))};
    HostMatchResult res[2];
    rc = e->match(st, 2, particle, true, huber_solver(1), 0.05, 0, res);   // one iteration each (:326, :334-339)
    if (rc != LAMA_OK) return rc;
    SE2 after[2] = {res[0].state, res[1].state};
    double err2[2];
    rc = e->match_error(after, 2, particle, true, err2);
    if (rc != LAMA_OK) return rc;
    const int pick = err2[0] < err2[1] ? 0 : 1;                            // :342-345
    HostMatchResult fin;
    rc = e->match(&after[pick], 1, particle, true, huber_solver(100), 0.05, 0, &fin);   // :348-349
    if (rc != LAMA_OK) return rc;
    rc = e->match_error(&fin.state, 1, particle, true, rmse);
    if (rc != LAMA_OK) return rc;
    *between = se2_mul(se2_inv(fin.state), ref_pose);                      // Pose2D(state) - ref_pose (:351, pose2d.cpp:81-84)
    return LAMA_OK;
}

int coarse_correlate_candidate_scan(Engine* e, int particle, const DeviceOptions& dev, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat,
                                    const double* pts, int n, const double* origin, const double* quat, const SE2& ref_pose, const SE2& cand_pose, SE2* between,
                                    double* rmse, std::string& err)
{
    // a coarse distance map of the reference cloud alone (:377-381): resolution 0.25 m, reach 2.5 m
    std::unique_ptr<DistanceMapDev> coarse(DistanceMapDev::create(0.25, 32, 2.5, ref_pose.tx, ref_pose.ty, dev, err));
    if (!coarse) return LAMA_ERR_CUDA;
    {
        ScanParams sp{};
        sp.n_beams = ref_n;
        sp.scale   = 1.0 / 0.25;
        Engine* ce = coarse->engine();
        int rc = ce->set_scan(ref_pts, ref_n, ref_origin, ref_quat, 0, 0);   // only to build the sensor transform exactly like the kernels do
        if (rc != LAMA_OK) { err = ce->last_error(); return rc; }
        const Affine tf = compose_tf(ref_pose, ce->scan_params().moving);
        std::vector<uint32_t> cells((size_t)ref_n * 2);
        for (int i = 0; i < ref_n; ++i) {
            double hit[3];
            apply_tf(tf, ref_pts[3 * i], ref_pts[3 * i + 1], ref_pts[3 * i + 2], hit);
            cells[2 * i]     = w2m(hit[0], sp.scale);
            cells[2 * i + 1] = w2m(hit[1], sp.scale);
        }
        rc = coarse->add(cells.data(), ref_n, true);
        uint32_t processed = 0;
        if (rc == LAMA_OK) rc = coarse->update(&processed);
        if (rc != LAMA_OK) { err = coarse->error(); return rc; }
        rc = ce->set_scan(pts, n, origin, quat, 0, 0);
        HostMatchResult r0;
        if (rc == LAMA_OK) rc = ce->match(&cand_pose, 1, 0, true, huber_solver(100), 0.05, 0, &r0);   // :383-384
        if (rc != LAMA_OK) { err = ce->last_error(); return rc; }
        int rc2 = e->set_scan(pts, n, origin, quat, 0, 0);
        HostMatchResult r1;
        if (rc2 == LAMA_OK) rc2 = e->match(&r0.state, 1, particle, true, huber_solver(100), 0.05, 0, &r1);   // :386-387
        if (rc2 == LAMA_OK) rc2 = e->match_error(&r1.state, 1, particle, true, rmse);
        if (rc2 != LAMA_OK) { err = e->last_error(); return rc2; }
        *between = se2_mul(se2_inv(r1.state), ref_pose);   // :389
    }
    return LAMA_OK;
}

// =====================================================================================================
// GraphSlam2D (src/graph_slam2d.cpp:104-430)
// =====================================================================================================
GraphSlam2D* GraphSlam2D::create(const GraphOptions& o, std::string& err)
{
    if (o.slam.lidar_odometry || o.slam.occupancy != 0) { err = "GraphSlam2D: the inner Slam2D runs on a FrequencyOccupancyMap without lidar odometry"; return nullptr; }
    GraphOptions g = o;
    g.slam.transient_map = true;   // :106-107
    g.slam.truncated_ray = 1.0;
    Slam2D* s = Slam2D::create(g.slam, err);
    if (!s) return nullptr;
    GraphSlam2D* gs = new GraphSlam2D();
    gs->opt_ = g;
    gs->slam_.reset(s);
    return gs;
}

int GraphSlam2D::update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double stamp, bool* did_update)
{
    *did_update = false;
    last_candidates_.clear();
    bool did = false;
    int rc = slam_->update(pts, n, origin, quat, odom_xyr, stamp, &did);   // 1. the transient slam (:193-195)
    if (rc != LAMA_OK) { err_ = slam_->error(); return rc; }
    if (!did) return LAMA_OK;
    *did_update = true;

    // 2. key pose test (:200-207): diff = slam pose - prev = pose^-1 prev
    const SE2 sp = slam_->pose();
    const SE2 diff = se2_mul(se2_inv(sp), prev_);
    if (xy_norm(diff) < opt_.key_pose_distance && std::fabs(se2_rotation(diff)) < opt_.key_pose_angular_distance) return LAMA_OK;
    prev_ = sp;

    // 4. the key pose and its factor (:210-228)
    int keyid = (int)keys_.size();
    const SE2 corrected = se2_mul(correction_, sp);
    if (keyid == 0) {
        priors_.push_back(PgoPrior{0, sp, PgoLoss{{0.01, 0.01, 0.01}, 0.0}});
    } else {
        accdist_ += xy_norm(diff);
        factors_.push_back(PgoBetween{keyid - 1, keyid, se2_mul(se2_inv(keys_.back().pose), corrected), PgoLoss{{0.25, 0.25, 0.15}, 0.0}});
    }
    KeyPose kp;
    kp.id = keyid;
    kp.pose = corrected;
    kp.original = sp;
    kp.pts.assign(pts, pts + 3 * (size_t)n);
    for (int k = 0; k < 3; ++k) kp.origin[k] = origin ? origin[k] : 0.0;
    for (int k = 0; k < 4; ++k) kp.quat[k] = quat ? quat[k] : (k == 3 ? 1.0 : 0.0);
    kp.stamp = stamp;
    keys_.push_back(std::move(kp));
    if (keyid < opt_.key_pose_head_delay || keyid < opt_.ignore_n_chain_poses) return LAMA_OK;   // :230-232

    // 5. loop closure search (:236-273): radius max^r min^(1 - r), query = the key pose head_delay keys back
    const double r = std::min(accdist_, 100.0) / 100.0;
    const double radius = std::pow(opt_.loop_search_max_distance, r) * std::pow(opt_.loop_search_min_distance, 1.0 - r);
    keyid -= opt_.key_pose_head_delay;
    std::vector<double> key_xy(keys_.size() * 2);
    for (size_t i = 0; i < keys_.size(); ++i) { key_xy[2 * i] = keys_[i].pose.tx; key_xy[2 * i + 1] = keys_[i].pose.ty; }
    const double query[2] = {keys_[(size_t)keyid].pose.tx, keys_[(size_t)keyid].pose.ty};
    last_candidates_ = find_loop_closure_candidates(key_xy.data(), (int)keys_.size(), opt_.ignore_n_chain_poses, query, radius, opt_.loop_max_candidates);
    factordist_ += xy_norm(diff);

    const SE2 cinv = se2_inv(correction_);
    const KeyPose& ref = keys_[(size_t)keyid];
    const SE2 ref_pose = se2_mul(cinv, ref.pose);   // Pose2D(correction.state.inverse()) + pose (:319-320)
    Engine* e = slam_->engine();
    for (size_t i = 0; i < last_candidates_.size(); ++i) {
        const int idx = last_candidates_[i];
        const KeyPose& cand = keys_[(size_t)idx];
        const SE2 cand_pose = se2_mul(cinv, cand.pose);
        SE2 between{1, 0, 0, 0};
        double rmse = 0.0;
        rc = correlate_candidate_scan(e, 0, cand.pts.data(), (int)(cand.pts.size() / 3), cand.origin, cand.quat, ref_pose, cand_pose, &between, &rmse);
        if (rc != LAMA_OK) { err_ = e->last_error(); return rc; }
        if (rmse > opt_.loop_closure_scan_rmse) {
            if (i != 0) continue;
            // one more chance, only for the closest candidate (:254-258)
            rc = coarse_correlate_candidate_scan(e, 0, slam_->device_options(), ref.pts.data(), (int)(ref.pts.size() / 3), ref.origin, ref.quat, cand.pts.data(),
                                                 (int)(cand.pts.size() / 3), cand.origin, cand.quat, ref_pose, cand_pose, &between, &rmse, err_);
            if (rc != LAMA_OK) return rc;
            if (rmse > opt_.loop_closure_scan_rmse * 2.0) continue;
        }
        links_.push_back({idx, keyid});                                              // :266-268, HuberLoss::Huber(0.1)
        queue_.push_back(PgoBetween{idx, keyid, between, PgoLoss{{1.0, 1.0, 1.0}, 0.1}});
        ++stats_.loop_factors;
        factordist_ = 0.0;
        break;   // only one factor per update
    }
    if (queue_.empty() || (queue_.size() <= 5 && factordist_ <= 15.0)) return LAMA_OK;   // :275-276
    rc = optimize_pose_graph();
    factordist_ = 0.0;
    return rc;
}

int GraphSlam2D::optimize_pose_graph()
{
    if (queue_.empty()) return LAMA_OK;
    factors_.insert(factors_.end(), queue_.begin(), queue_.end());   // :399-402
    queue_.clear();
    std::vector<SE2> nodes(keys_.size());
    for (size_t i = 0; i < keys_.size(); ++i) nodes[i] = keys_[i].pose;   // :408-411
    PgoReport rep;
    std::string e;
    int rc = pgo_optimize_graph(opt_.slam.dev.device, nodes, priors_, factors_, rep, e);   // LevenbergMarquardtOptimizer, default parameters (:404-413)
    if (rc != LAMA_OK) { err_ = e; return rc; }
    ++stats_.optimizations;
    if (rep.status == 0) {   // :414-426: propagate the corrections, correction = (B A^-1)^-1
        ++stats_.optimizations_ok;
        for (size_t i = 0; i < keys_.size(); ++i) keys_[i].pose = nodes[i];
        correction_ = se2_inv(se2_mul(slam_->pose(), se2_inv(keys_.back().pose)));
    }
    stats_.last = std::move(rep);
    mapping_keyid_ = 0;   // :428-429
    accdist_ = 0.0;
    return LAMA_OK;
}

// the inner Slam2D's window centre (its engine is created at the first update, centred on the pose of that moment)
static void slam_window_center(Slam2D* s, double c[2])
{
    if (s->engine()) {
        c[0] = s->engine()->config().center_x;
        c[1] = s->engine()->config().center_y;
    } else {
        c[0] = s->pose().tx;
        c[1] = s->pose().ty;
    }
}

int GraphSlam2D::generate_occupancy_map(bool full, OccupancyMapDev** out)
{
    if (mapping_keyid_ == 0 || !occ_) {   // :132-133
        double c[2];
        slam_window_center(slam_.get(), c);
        OccupancyMapDev* m = OccupancyMapDev::create(full ? opt_.slam.resolution : 0.1, 32, c[0], c[1], slam_->device_options(), err_);
        if (!m) return LAMA_ERR_CUDA;
        occ_.reset(m);   // borrowed handles never see a null map
        mapping_keyid_ = 0;
    }
    const size_t n_scans = keys_.size() - mapping_keyid_;
    std::vector<double> pts, origins, quats;
    std::vector<int64_t> offsets(1, 0);
    std::vector<SE2> states;
    for (size_t i = mapping_keyid_; i < keys_.size(); ++i) {   // :135-160, the key's CURRENT (corrected) pose
        const KeyPose& k = keys_[i];
        pts.insert(pts.end(), k.pts.begin(), k.pts.end());
        offsets.push_back(offsets.back() + (int64_t)(k.pts.size() / 3));
        origins.insert(origins.end(), k.origin, k.origin + 3);
        quats.insert(quats.end(), k.quat, k.quat + 4);
        states.push_back(k.pose);
    }
    int rc = occ_->insert_scans(pts.data(), offsets.data(), (int)n_scans, origins.data(), quats.data(), states.data(), full, nullptr);
    if (rc == LAMA_OK) rc = occ_->prune();   // :162
    if (rc != LAMA_OK) { err_ = occ_->error(); return rc; }
    mapping_keyid_ = keys_.size();           // :163
    *out = occ_.get();
    return LAMA_OK;
}

int GraphSlam2D::generate_coarse_distance_map(DistanceMapDev** out, uint32_t* processed)
{
    Engine* e = slam_->engine();
    if (!e) { err_ = "no map yet (update() has not been called)"; return LAMA_ERR_STATE; }
    double c[2];
    slam_window_center(slam_.get(), c);
    // visit_all_cells of the inner distance map (:171): its known cells are those of its own patches and, for a frequency map, every
    // touched occupancy cell (see unpack_distance_words); both maps are read over the union of their patches
    uint32_t a0[2], a1[2], b0[2], b1[2];
    const int nd = e->bounds(0, 1, a0, a1), no = e->bounds(0, 0, b0, b1);
    if (nd < 0 || no < 0) { err_ = e->last_error(); return LAMA_ERR_ARG; }
    std::vector<uint32_t> cells;
    std::unordered_set<uint64_t> seen;
    if (nd + no > 0) {
        uint32_t mn[2], mx[2];
        for (int k = 0; k < 2; ++k) {
            mn[k] = nd && no ? std::min(a0[k], b0[k]) : (nd ? a0[k] : b0[k]);
            mx[k] = nd && no ? std::max(a1[k], b1[k]) : (nd ? a1[k] : b1[k]);
        }
        const int w = (int)(mx[0] - mn[0]), h = (int)(mx[1] - mn[1]);
        std::vector<uint32_t> dw((size_t)w * h), ow((size_t)w * h);
        int rc = e->export_window(0, 1, mn[0], mn[1], w, h, dw.data(), nullptr);
        if (rc == LAMA_OK) rc = e->export_window(0, 0, mn[0], mn[1], w, h, ow.data(), nullptr);
        if (rc != LAMA_OK) { err_ = e->last_error(); return rc; }
        const double fine = 1.0 / opt_.slam.resolution, coarse = 1.0 / 0.1;
        // ascending directory index = patch rows bottom up, patches left to right; then cells in container order (x fastest)
        for (int py = 0; py < h; py += kPatchLen)
            for (int px = 0; px < w; px += kPatchLen)
                for (int y = py; y < py + kPatchLen; ++y)
                    for (int x = px; x < px + kPatchLen; ++x) {
                        const size_t i = (size_t)y * w + x;
                        const bool known = (dw[i] & kDmKnown) || ow[i] != 0;
                        if (!known || !occ_is_occupied(occ_occupied(ow[i]), occ_visited(ow[i]))) continue;   // isOccupied (:173-174)
                        uint32_t m[2];
                        for (int k = 0; k < 2; ++k) {
                            const double wpos = ((double)((k ? mn[1] + (uint32_t)y : mn[0] + (uint32_t)x)) - (double)kMapOffsetCells) / fine;   // m2w (map.h:147-148)
                            m[k] = w2m(wpos, coarse);                                                                                      // w2m (:176)
                        }
                        // a repeated addObstacle of a cell is a no-op (dynamic_distance_map.cpp:217-218): only the first call is kept, so the
                        // list stays within one brushfire batch
                        if (!seen.insert((uint64_t)m[0] << 32 | m[1]).second) continue;
                        cells.push_back(m[0]);
                        cells.push_back(m[1]);
                    }
    }
    // :168-169; the whole list goes through one brushfire, as the reference's single update() (lists beyond 8 192 cells are applied in
    // batches, DESIGN.md 10)
    const int n = (int)(cells.size() / 2);
    DistanceMapDev* dm = DistanceMapDev::create(0.1, 32, 5.0, c[0], c[1], slam_->device_options(), err_, std::min(n, 8192));
    if (!dm) return LAMA_ERR_CUDA;
    coarse_dm_.reset(dm);   // borrowed handles never see a null map
    int rc = dm->add(cells.data(), n, true);
    if (rc == LAMA_OK) rc = dm->update(processed);   // :183
    if (rc != LAMA_OK) { err_ = dm->error(); return rc; }
    *out = dm;
    return LAMA_OK;
}

// =====================================================================================================
// Slam2D
// =====================================================================================================
Slam2D* Slam2D::create(const SlamOptions& o, std::string& err)
{
    if (o.patch_size != 32) { err = "Slam2D: only patch_size 32 is supported on the device"; return nullptr; }
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    Slam2D* s = new Slam2D();
    s->opt_ = o;
    return s;
}

int Slam2D::update_maps(const double* pts, int n)
{
    HostMapStats st{};
    int rc = eng_->update_maps(&pose_, 0, 1, &st);
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    processed_ = st.dm_pops;  // number_of_proccessed_cells_, slam2d.cpp:321
    last_.ray_cells = st.ray_cells;
    last_.dm_pops   = st.dm_pops;
    total_.add(last_);
    ++map_updates_;
    if (!opt_.transient_map && !opt_.lidar_odometry) return LAMA_OK;
    // Transient map (slam2d.cpp:323-379; lidar_odometry_2d.cpp:130-181 without the factor 2): the surface AABB comes from the world
    // hits of this scan (the same expression the kernel evaluates per beam), the patch test and the deletion run on the device maps.
    const ScanParams& sp = eng_->scan_params();
    const Affine tf = compose_tf(pose_, sp.moving);
    double mn[2] = {std::numeric_limits<double>::max(), std::numeric_limits<double>::max()}, mx[2] = {-mn[0], -mn[1]};
    for (int i = 0; i < n; ++i) {
        double hit[3], start[3];
        beam_world(tf, sp, pts + 3 * (size_t)i, hit, start);
        for (int k = 0; k < 2; ++k) { mn[k] = std::min(mn[k], hit[k]); mx[k] = std::max(mx[k], hit[k]); }
    }
    const double stretch = opt_.lidar_odometry ? 1.0 : 2.0;
    const double xdist = std::max(pose_.tx - mn[0], mx[0] - pose_.tx) * stretch, ydist = std::max(pose_.ty - mn[1], mx[1] - pose_.ty) * stretch;
    mn[0] = pose_.tx - xdist; mn[1] = pose_.ty - ydist;
    mx[0] = pose_.tx + xdist; mx[1] = pose_.ty + ydist;
    double center[2], hwidth[2];
    const double reach = std::sqrt((double)eng_->max_sqdist()) * opt_.resolution;   // DistanceMap::maxDistance, dynamic_distance_map.cpp:155-158
    for (int k = 0; k < 2; ++k) {
        hwidth[k] = (mx[k] - mn[k]) * 0.5;           // AABB(min, max), aabb.h:50-55
        center[k] = mn[k] + hwidth[k];
        hwidth[k] += 2.0 * reach;
    }
    int removed = 0;
    rc = eng_->prune_outside(0, center, hwidth, &removed);
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    removed_ += (uint64_t)removed;
    return LAMA_OK;
}

// LidarOdometry2D::update (lidar_odometry_2d.cpp:59-83)
int Slam2D::update_lidar_odometry(const double* pts, int n, const double* origin, const double* quat, bool* did_update)
{
    int rc = eng_->set_scan(pts, n, origin, quat, 0.0, 0.0);
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    *did_update = true;
    if (!has_first_) {
        rc = update_maps(pts, n);
        has_first_ = true;
        return rc;
    }
    HostMatchResult res;
    rc = eng_->match(&pose_, 1, 0, false, make_solver(0, opt_.max_iter), 0.05, 0, &res);   // GaussNewton + CauchyWeight(0.15), :48-50
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    pose_ = res.state;
    last_.evals    = res.evals_ref;
    last_.gn_iters = res.iterations;
    const SE2 odelta = se2_mul(se2_inv(map_update_pose_), pose_);   // map_update_odom - odom (pose2d.cpp:81-84)
    if (xy_norm(odelta) > 0.1 || std::abs(se2_rotation(odelta)) > 0.5) {
        rc = update_maps(pts, n);
        map_update_pose_ = pose_;
        return rc;
    }
    total_.add(last_);
    return LAMA_OK;
}

int Slam2D::update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double, bool* did_update)
{
    *did_update = false;
    last_ = Counters();
    if (!eng_) {
        std::string e;
        if (opt_.lidar_odometry) {   // lidar_odometry_2d.cpp:44-46
            opt_.l2_max    = 1.0;
            opt_.occupancy = 1;
        }
        EngineConfig cfg = engine_config(opt_.dev, 1, opt_.resolution, opt_.l2_max, pose_.tx, pose_.ty);
        cfg.max_beams = std::max(cfg.max_beams, n);
        cfg.occupancy_kind = opt_.occupancy == 1 ? 1 : 0;
        Engine* en = Engine::create(cfg, e);
        if (!en) { err_ = e; return LAMA_ERR_CUDA; }
        eng_.reset(en);
        eng_->enable_timing(opt_.dev.timing != 0);
        eng_->set_lidar_odometry_rays(opt_.lidar_odometry);
    }
    if (opt_.lidar_odometry) return update_lidar_odometry(pts, n, origin, quat, did_update);
    if (!odom_xyr) { err_ = "Slam2D::update needs an odometry pose"; return LAMA_ERR_ARG; }
    const SE2 odometry = se2_from_xyr(odom_xyr[0], odom_xyr[1], odom_xyr[2]);
    if (!has_first_) {  // slam2d.cpp:147-161
        int rc = eng_->set_scan(pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range);
        if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
        odom_ = odometry;
        rc = update_maps(pts, n);
        if (rc != LAMA_OK) return rc;
        has_first_  = true;
        *did_update = true;
        return LAMA_OK;
    }
    const SE2 odelta = se2_mul(se2_inv(odom_), odometry);
    const SE2 ppose  = se2_mul(pose_, odelta);
    if (xy_norm(odelta) <= opt_.trans_thresh && std::abs(se2_rotation(odelta)) <= opt_.rot_thresh) return LAMA_OK;  // slam2d.cpp:168-170
    pose_ = ppose;
    odom_ = odometry;
    int rc = eng_->set_scan(pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range);
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    HostMatchResult res;
    rc = eng_->match(&pose_, 1, 0, false, make_solver(opt_.strategy, opt_.max_iter), 0.05, 0, &res);
    if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    pose_ = res.state;
    last_.evals    = res.evals_ref;
    last_.gn_iters = res.iterations;
    *did_update = true;
    return update_maps(pts, n);
}

// =====================================================================================================
// DistanceMapDev + Loc2D
// =====================================================================================================
DistanceMapDev* DistanceMapDev::create(double resolution, uint32_t patch_size, double l2_max, double cx, double cy, const DeviceOptions& dev,
                                       std::string& err, int event_cap)
{
    if (patch_size != 32) { err = "DynamicDistanceMap: only patch_size 32 is supported on the device"; return nullptr; }
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    EngineConfig cfg = engine_config(dev, 1, resolution, l2_max, cx, cy);
    cfg.event_cap = event_cap;
    Engine* en = Engine::create(cfg, err);
    if (!en) return nullptr;
    DistanceMapDev* d = new DistanceMapDev();
    d->eng_.reset(en);
    en->enable_timing(dev.timing != 0);
    return d;
}

int DistanceMapDev::add(const uint32_t* cells_xy, int n, bool is_add)
{
    // addObstacle / removeObstacle only mark cells and queue them; they take effect on the device at
    // the next update() in call order (the reference's queues are drained by update() as well).
    for (int i = 0; i < n; ++i) {
        pend_cells_.push_back(cells_xy[2 * i]);
        pend_cells_.push_back(cells_xy[2 * i + 1]);
        pend_kind_.push_back(is_add ? 1 : 0);
    }
    return LAMA_OK;
}

int DistanceMapDev::update(uint32_t* processed)
{
    uint32_t p = 0;
    int rc = eng_->dm_apply(0, pend_cells_.data(), pend_kind_.data(), (int)pend_kind_.size(), &p);
    pend_cells_.clear();
    pend_kind_.clear();
    if (rc != LAMA_OK) err_ = eng_->last_error();
    if (processed) *processed = p;
    return rc;
}

int DistanceMapDev::flush_if_pending()
{
    if (pend_kind_.empty()) return LAMA_OK;
    // Reads of a map with queued-but-unpropagated obstacle changes see the marked cells in the
    // reference; here the marks are applied lazily, so bring the device up to date first.
    return update(nullptr);
}

OccupancyMapDev* OccupancyMapDev::create(double resolution, uint32_t patch_size, double cx, double cy, const DeviceOptions& dev, std::string& err)
{
    if (patch_size != 32) { err = "FrequencyOccupancyMap: only patch_size 32 is supported on the device"; return nullptr; }
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    EngineConfig cfg = engine_config(dev, 1, resolution, resolution, cx, cy);   // no distance map is kept: the smallest reach
    if (cfg.pool_slots <= 0) cfg.pool_slots = cfg.dir_dim * cfg.dir_dim;
    cfg.known_plane = true;
    Engine* en = Engine::create(cfg, err);
    if (!en) return nullptr;
    OccupancyMapDev* m = new OccupancyMapDev();
    m->eng_.reset(en);
    en->enable_timing(dev.timing != 0);
    return m;
}

OccupancyMapDev* OccupancyMapDev::adopt(Engine* e)
{
    OccupancyMapDev* m = new OccupancyMapDev();
    m->eng_.reset(e);
    return m;
}

int OccupancyMapDev::insert_scans(const double* pts, const int64_t* offsets, int n_scans, const double* origins, const double* quats, const SE2* states,
                                  bool full, uint64_t* cells)
{
    int rc = eng_->render_scans(pts, offsets, n_scans, origins, quats, states, full, cells);
    if (rc != LAMA_OK) err_ = eng_->last_error();
    return rc;
}

int OccupancyMapDev::prune()
{
    int rc = eng_->prune_frequency();
    if (rc != LAMA_OK) err_ = eng_->last_error();
    return rc;
}

// ---- SimpleOccupancyHost ---------------------------------------------------------------------------------------
void SimpleOccupancyHost::set(uint32_t x, uint32_t y, int state)
{
    const uint64_t key = (uint64_t)(x >> kPatchLog2) * 2642244ull + (uint64_t)(y >> kPatchLog2);  // Map::m2p, map.h:153-161
    auto it = patches_.find(key);
    if (it == patches_.end()) it = patches_.emplace(key, std::vector<int8_t>(kPatchCells, 0)).first;
    it->second[cell_index(x, y)] = (int8_t)(state < 0 ? -1 : (state > 0 ? 1 : 0));
}
bool SimpleOccupancyHost::is_free_world(double wx, double wy) const
{
    const uint32_t x = w2m(wx, scale_), y = w2m(wy, scale_);
    auto it = patches_.find((uint64_t)(x >> kPatchLog2) * 2642244ull + (uint64_t)(y >> kPatchLog2));
    return it != patches_.end() && it->second[cell_index(x, y)] == -1;
}
bool SimpleOccupancyHost::bounds_world(double mn[2], double mx[2]) const
{
    if (patches_.empty()) return false;
    uint32_t lo[2] = {0xffffffffu, 0xffffffffu}, hi[2] = {0, 0};
    for (auto& kv : patches_) {
        const uint32_t ax = (uint32_t)(kv.first / 2642244ull) << kPatchLog2, ay = (uint32_t)(kv.first % 2642244ull) << kPatchLog2;  // Map::p2m
        lo[0] = std::min(lo[0], ax); lo[1] = std::min(lo[1], ay);
        hi[0] = std::max(hi[0], ax); hi[1] = std::max(hi[1], ay);
    }
    for (int k = 0; k < 2; ++k) {
        mn[k] = ((double)lo[k] - (double)kMapOffsetCells) / scale_;               // Map::m2w
        mx[k] = ((double)(hi[k] + kPatchLen) - (double)kMapOffsetCells) / scale_;
    }
    return true;
}

Loc2D* Loc2D::create(const LocOptions& o, std::string& err)
{
    DistanceMapDev* dm = DistanceMapDev::create(o.resolution, o.patch_size, o.l2_max, o.center_x, o.center_y, o.dev, err);
    if (!dm) return nullptr;
    Loc2D* l = new Loc2D();
    l->opt_ = o;
    l->dm_.reset(dm);
    l->occ_.reset(new SimpleOccupancyHost(o.resolution));
    l->cov_blend_ = std::max(std::min(o.cov_blend, 1.0), 0.0);  // loc2d.cpp:90
    const double sstep = o.resolution;                           // loc2d.cpp:93-107
    auto add = [&](double x, double y) { l->sampling_steps_.push_back(x); l->sampling_steps_.push_back(y); };
    add(0.0, 0.0);
    for (int i = 1; i <= 20; ++i) {
        add(i * sstep, 0.0); add(0.0, i * sstep); add(-i * sstep, 0.0); add(0.0, -i * sstep);
        add(i * sstep, i * sstep); add(-i * sstep, i * sstep); add(i * sstep, -i * sstep); add(-i * sstep, -i * sstep);
    }
    return l;
}

// Loc2D::globalLocalization (loc2d.cpp:249-286): candidates are drawn on the host with the reference's rejection
// sampling (same generator calls in the same order), evaluated in ONE device launch (the same evaluation kernel as
// scan matching, every block on the same map) and the best is chosen with the reference's strict `<` in index order.
int Loc2D::global_localization(int n)
{
    double mn[2], mx[2];
    if (!occ_->bounds_world(mn, mx)) return LAMA_OK;
    const double diff[2] = {mx[0] - mn[0], mx[1] - mn[1]};
    std::vector<SE2> cand(opt_.gloc_particles);
    auto uniform = [&]() { std::uniform_real_distribution<double> d(0.0, 1.0); return d(gen_); };
    for (uint32_t i = 0; i < opt_.gloc_particles; ++i) {
        double x, y, a;
        for (;;) {
            x = mn[0] + uniform() * diff[0];
            y = mn[1] + uniform() * diff[1];
            if (!occ_->is_free_world(x, y)) continue;
            a = uniform() * 2 * M_PI - M_PI;
            break;
        }
        cand[i] = se2_from_xyr(x, y, a);
    }
    std::vector<HostMatchResult> res(cand.size());
    SolverOptions so = make_solver(0, 0);
    int rc = dm_->engine()->match(cand.data(), (int)cand.size(), 0, true, so, 0.05, 1, res.data());
    if (rc != LAMA_OK) { err_ = dm_->engine()->last_error(); return rc; }
    double best = std::numeric_limits<double>::max();
    for (size_t i = 0; i < cand.size(); ++i)
        if (res[i].sums[10] < best) {  // residuals.squaredNorm()
            best  = res[i].sums[10];
            pose_ = cand[i];
        }
    (void)n;
    return LAMA_OK;
}

// Loc2D::addSamplingCovariance (loc2d.cpp:199-247)
int Loc2D::add_sampling_covariance(int n)
{
    const int n_off = (int)(sampling_steps_.size() / 2);
    const int stride = (int)std::max((size_t)n / 100, (size_t)1);
    std::vector<double> l((size_t)n_off);
    int rc = dm_->engine()->sampling_likelihood(0, pose_, sampling_steps_.data(), n_off, stride, l.data());
    if (rc != LAMA_OK) { err_ = dm_->engine()->last_error(); return rc; }
    double K[4] = {0, 0, 0, 0}, u[2] = {0, 0}, sl = 0;
    for (int i = 0; i < n_off; ++i) {
        const double x = pose_.tx + sampling_steps_[2 * i], y = pose_.ty + sampling_steps_[2 * i + 1];
        K[0] = K[0] + x * x * l[i]; K[1] = K[1] + x * y * l[i]; K[2] = K[2] + y * x * l[i]; K[3] = K[3] + y * y * l[i];
        u[0] = u[0] + x * l[i]; u[1] = u[1] + y * l[i];
        sl = sl + l[i];
    }
    const double a = 1.0 / sl, b = 1.0 / (sl * sl);
    const double sc[4] = {a * K[0] - b * u[0] * u[0], a * K[1] - b * u[0] * u[1], a * K[2] - b * u[1] * u[0], a * K[3] - b * u[1] * u[1]};
    const double alpha = cov_blend_;
    cov_[0] = alpha * sc[0] + (1.0 - alpha) * cov_[0]; cov_[1] = alpha * sc[1] + (1.0 - alpha) * cov_[1];
    cov_[3] = alpha * sc[2] + (1.0 - alpha) * cov_[3]; cov_[4] = alpha * sc[3] + (1.0 - alpha) * cov_[4];
    return LAMA_OK;
}

// Solver::calculateCovariance (solver.cpp:133-150): (J^T J)^-1 when J has full column rank, else the
// thin-SVD pseudo inverse V diag(f(sv)) V^T with f = 1/sv^2 for |sv| > 1e-3 and 3.0 otherwise.
void covariance_from_sums(const double s[kNumSums], size_t rows, double cov[9])
{
    const double A[9] = {s[0], s[1], s[2], s[1], s[3], s[4], s[2], s[4], s[5]};
    // Jacobi eigen-decomposition of the symmetric 3x3
    double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) a[i][j] = A[i * 3 + j];
    for (int sweep = 0; sweep < 64; ++sweep) {
        double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (a[p][q] == 0.0) continue;
                double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
                double t = ((theta >= 0) ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                double c = 1.0 / std::sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < 3; ++k) { double akp = a[k][p], akq = a[k][q]; a[k][p] = c * akp - sn * akq; a[k][q] = sn * akp + c * akq; }
                for (int k = 0; k < 3; ++k) { double apk = a[p][k], aqk = a[q][k]; a[p][k] = c * apk - sn * aqk; a[q][k] = sn * apk + c * aqk; }
                for (int k = 0; k < 3; ++k) { double vkp = v[k][p], vkq = v[k][q]; v[k][p] = c * vkp - sn * vkq; v[k][q] = sn * vkp + c * vkq; }
            }
    }
    double w[3] = {a[0][0], a[1][1], a[2][2]};
    const double wmax = std::max(w[0], std::max(w[1], w[2])), wmin = std::min(w[0], std::min(w[1], w[2]));
    const double thr  = 2.220446049250313e-16 * (double)std::max<size_t>(rows, 3);
    const bool full   = wmax > 0 && std::sqrt(std::max(wmin, 0.0)) > thr * std::sqrt(wmax);
    if (full) {
        // Gauss-Jordan with partial pivoting
        double M[3][6];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { M[i][j] = A[i * 3 + j]; M[i][3 + j] = (i == j) ? 1.0 : 0.0; }
        bool ok = true;
        for (int k = 0; k < 3 && ok; ++k) {
            int piv = k;
            for (int i = k + 1; i < 3; ++i) if (std::fabs(M[i][k]) > std::fabs(M[piv][k])) piv = i;
            if (M[piv][k] == 0.0) { ok = false; break; }
            if (piv != k) for (int j = 0; j < 6; ++j) std::swap(M[k][j], M[piv][j]);
            double d = M[k][k];
            for (int j = 0; j < 6; ++j) M[k][j] /= d;
            for (int i = 0; i < 3; ++i) {
                if (i == k) continue;
                double f = M[i][k];
                for (int j = 0; j < 6; ++j) M[i][j] -= f * M[k][j];
            }
        }
        if (ok) {
            for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) cov[i * 3 + j] = M[i][3 + j];
            return;
        }
    }
    double f[3];
    for (int i = 0; i < 3; ++i) {
        double sv = std::sqrt(std::max(w[i], 0.0));
        f[i] = (std::fabs(sv) > 1.e-3) ? 1.0 / (sv * sv) : 3.0;
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double acc = 0;
            for (int k = 0; k < 3; ++k) acc += v[i][k] * f[k] * v[j][k];
            cov[i * 3 + j] = acc;
        }
}

int Loc2D::update(const double* pts, int n, const double* origin, const double* quat, const double odom_xyr[3], double, bool force, bool* did_update)
{
    *did_update = false;
    Engine* eng = dm_->engine();
    int rc = dm_->flush_if_pending();
    if (rc != LAMA_OK) { err_ = dm_->error(); return rc; }
    const SE2 odometry = se2_from_xyr(odom_xyr[0], odom_xyr[1], odom_xyr[2]);
    SolverOptions so = make_solver(opt_.strategy, opt_.max_iter);
    bool scan_set = false;
    if (!has_first_) {  // loc2d.cpp:128-141
        odom_      = odometry;
        has_first_ = true;
        if (!force) { *did_update = true; return LAMA_OK; }
        rc = eng->set_scan(pts, n, origin, quat, 0, 0);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
        scan_set = true;
        HostMatchResult r;
        rc = eng->match(&pose_, 1, 0, false, so, 0.05, 1, &r);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
        rmse_ = std::sqrt(r.sums[10] / ((double)((size_t)n - 1)));
    }
    const SE2 odelta = se2_mul(se2_inv(odom_), odometry);
    const SE2 ppose  = se2_mul(pose_, odelta);
    const bool enough = !(xy_norm(odelta) <= opt_.trans_thresh && std::abs(se2_rotation(odelta)) <= opt_.rot_thresh);
    if (!force && !enough) return LAMA_OK;
    pose_ = ppose;
    odom_ = odometry;
    if (!scan_set) {
        rc = eng->set_scan(pts, n, origin, quat, 0, 0);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
    }
    if (do_gloc_) {  // loc2d.cpp:154-166
        if (gloc_cur_iter_ < opt_.gloc_iters) {
            gloc_cur_iter_++;
            rc = global_localization(n);
            if (rc != LAMA_OK) return rc;
        } else {
            do_gloc_       = false;
            gloc_cur_iter_ = 0;
        }
    }
    HostMatchResult r;
    rc = eng->match(&pose_, 1, 0, false, so, 0.05, 0, &r);
    if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
    pose_  = r.state;
    iters_ = r.iterations;
    evals_ = r.evals_ref + 2;  // + the covariance and rmse evaluations of solver.cpp:110 / loc2d.cpp:178
    covariance_from_sums(r.sums, (size_t)n, cov_);
    if (cov_blend_ > 0.0) {     // loc2d.cpp:175-176
        rc = add_sampling_covariance(n);
        if (rc != LAMA_OK) return rc;
    }
    rmse_ = std::sqrt(r.sums[10] / ((double)((size_t)n - 1)));  // loc2d.cpp:178-180
    if (do_gloc_ && rmse_ < opt_.gloc_thresh) {                 // loc2d.cpp:182-188
        do_gloc_       = false;
        gloc_cur_iter_ = 0;
    }
    *did_update = true;
    return LAMA_OK;
}

void unpack_distance_words(const uint32_t* words, const uint8_t* occ_known, size_t n, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                           int16_t* oy, uint8_t* queued)
{
    for (size_t i = 0; i < n; ++i) {
        const uint32_t w = words[i];
        if (sqdist) sqdist[i] = (uint16_t)dm_sqdist(w);
        if (valid) valid[i] = (w & kDmValid) ? 1 : 0;
        if (known) known[i] = ((w & kDmKnown) || (occ_known && occ_known[i])) ? 1 : 0;
        if (ox) ox[i] = (int16_t)dm_ox(w);
        if (oy) oy[i] = (int16_t)dm_oy(w);
        if (queued) queued[i] = (w & kDmQueued) ? 1 : 0;
    }
}

// =====================================================================================================
// Checkpoints (format: checkpoint.h, DESIGN.md §13)
// =====================================================================================================
namespace {
using clk = std::chrono::steady_clock;
double ms_since(clk::time_point a) { return std::chrono::duration<double, std::milli>(clk::now() - a).count(); }

void put_counters(CkptWriter& w, const Counters& c)
{
    w.u64(c.evals); w.u64(c.ray_cells); w.u64(c.dm_pops); w.u64(c.detached); w.u64(c.gn_iters); w.u64(c.resampled);
}
Counters get_counters(CkptReader& r)
{
    Counters c;
    c.evals = r.u64("counters"); c.ray_cells = r.u64("counters"); c.dm_pops = r.u64("counters");
    c.detached = r.u64("counters"); c.gn_iters = r.u64("counters"); c.resampled = r.u64("counters");
    return c;
}
void put_geometry(CkptWriter& w, const DeviceOptions& d) { w.i32(d.dir_dim); w.i32(d.pool_slots); w.i32(d.max_beams); }
void get_geometry(CkptReader& r, DeviceOptions& d) { d.dir_dim = r.i32("dir_dim"); d.pool_slots = r.i32("pool_slots"); d.max_beams = r.i32("max_beams"); }
// the caller's dir_dim / pool_slots / max_beams: 0, or the file's (its options, or the engine it holds)
bool geometry_matches(const DeviceOptions& call, const DeviceOptions& file, const EngineImage* img, std::string& err)
{
    auto ok = [](int v, int opt, int eng) { return v == 0 || v == opt || v == eng; };
    if (ok(call.dir_dim, file.dir_dim, img ? img->dir_dim : file.dir_dim) && ok(call.pool_slots, file.pool_slots, img ? img->pool_slots : file.pool_slots) &&
        ok(call.max_beams, file.max_beams, img ? img->max_beams : file.max_beams))
        return true;
    err = "device options differ from the checkpoint's geometry (dir_dim, pool_slots and max_beams must be 0 or the saved values)";
    return false;
}
bool finite_se2(const SE2& s) { return std::isfinite(s.c) && std::isfinite(s.s) && std::isfinite(s.tx) && std::isfinite(s.ty); }
uint64_t sum_refs(const EngineImage& img)
{
    uint64_t n = 0;
    for (int32_t v : img.refcount) n += (uint64_t)v;
    return n;
}
// the refusal of a loader called on another handle kind's file
std::string wrong_kind(uint32_t kind, const char* want)
{
    const char* held = kind == kCkptPFSlam2D ? "PFSlam2D"
                       : kind == kCkptSlam2D || kind == kCkptLidarOdometry2D ? "Slam2D"
                       : kind == kCkptGraphSlam2D ? "GraphSlam2D" : nullptr;
    return held ? std::string("the checkpoint holds a ") + held + ", not a " + want : std::string("unknown checkpoint handle kind");
}
void add_times(CheckpointTimes& a, const CheckpointTimes& b)
{
    a.count_ms += b.count_ms; a.compact_ms += b.compact_ms; a.gather_ms += b.gather_ms;
    a.copy_ms += b.copy_ms; a.create_ms += b.create_ms; a.tables_ms += b.tables_ms;
}
}  // namespace

int PFSlam2D::save(const std::string& path, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    if (opt_.shard_count > 1) return fail("saveState: a sharded handle cannot be saved (each rank holds only its part of the filter)", LAMA_ERR_STATE);
    EngineImage img;
    if (eng_) {
        int rc = settle_counters();   // the pending map update and its counters, as the getters would book them
        if (rc != LAMA_OK) return rc;
        rc = eng_->snapshot(&img, &s.dev);
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    const auto t1 = clk::now();
    CkptWriter w;
    // options
    w.u32(opt_.particles);
    for (double v : {opt_.srr, opt_.str, opt_.stt, opt_.srt, opt_.meas_sigma, opt_.meas_sigma_gain, opt_.trans_thresh, opt_.rot_thresh, opt_.l2_max,
                     opt_.truncated_ray, opt_.truncated_range, opt_.resolution})
        w.f64(v);
    w.u32(opt_.patch_size); w.u32(opt_.max_iter); w.i32(opt_.strategy); w.i32(opt_.threads); w.u32(opt_.seed);
    put_geometry(w, opt_.dev);
    // front-end state
    w.se2(prior_); w.se2(odom_); w.u8(has_first_);
    w.f64(acc_trans_); w.f64(acc_rot_); w.f64(neff_);
    for (uint32_t i = 0; i < P_; ++i) w.se2(pose_[i]);
    for (const std::vector<double>* v : {&weight_, &nweight_, &wsum_}) w.bytes(v->data(), (size_t)P_ * 8);
    w.u32((uint32_t)last_idx_.size());
    w.bytes(last_idx_.data(), last_idx_.size() * 4);
    w.u64(resample_count_); w.u64(resample_hash_); w.u64(scans_seen_);
    w.u32((uint32_t)timestamps_.size());
    w.bytes(timestamps_.data(), timestamps_.size() * 8);
    put_counters(w, last_); put_counters(w, total_);
    w.u64(detached_seen_);
    w.f64(t_sample_); w.f64(t_solve_); w.f64(t_norm_); w.f64(t_resample_);
    // the trajectory nodes reachable from the particles, renumbered in their old order (a parent precedes its children)
    std::vector<int> renum(nodes_.size(), -1);
    for (uint32_t i = 0; i < P_; ++i)
        for (int n = node_of_[i]; n >= 0 && renum[(size_t)n] < 0; n = nodes_[(size_t)n].parent) renum[(size_t)n] = 0;
    uint32_t kept = 0;
    for (int& v : renum)
        if (v == 0) v = (int)kept++;
    w.u32(kept);
    for (size_t n = 0; n < nodes_.size(); ++n)
        if (renum[n] >= 0) {
            w.se2(nodes_[n].pose);
            w.i32(nodes_[n].parent < 0 ? -1 : renum[(size_t)nodes_[n].parent]);
        }
    for (uint32_t i = 0; i < P_; ++i) w.i32(node_of_[i] < 0 ? -1 : renum[(size_t)node_of_[i]]);
    std::ostringstream rng;
    rng << gen_;
    w.str(rng.str());
    ckpt_put_engine(w, eng_ ? &img : nullptr);
    s.encode_ms = ms_since(t1);
    std::string err;
    const int rc = ckpt_write_file(path, kCkptPFSlam2D, w, {{img.slot_bytes, (size_t)img.used * img.slot_stride()}}, err, &s);
    if (rc != LAMA_OK) return fail(err, rc);
    s.used_slots = img.used;
    s.references = sum_refs(img);
    s.total_ms   = ms_since(t0);
    return LAMA_OK;
}

PFSlam2D* PFSlam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    std::vector<uint8_t> file;
    uint32_t kind = 0;
    *code = ckpt_read_file(path, file, &kind, err, &s);
    if (*code != LAMA_OK) return nullptr;
    *code = LAMA_ERR_ARG;
    if (kind != kCkptPFSlam2D) {
        err = wrong_kind(kind, "PFSlam2D");
        return nullptr;
    }
    const auto t1 = clk::now();
    CkptReader r(file.data() + kCkptHeaderBytes, file.size() - kCkptHeaderBytes);
    PFOptions o;
    o.particles = r.u32("options");
    double* f[] = {&o.srr, &o.str, &o.stt, &o.srt, &o.meas_sigma, &o.meas_sigma_gain, &o.trans_thresh, &o.rot_thresh, &o.l2_max, &o.truncated_ray,
                   &o.truncated_range, &o.resolution};
    for (double* v : f) *v = r.f64("options");
    o.patch_size = r.u32("options"); o.max_iter = r.u32("options"); o.strategy = r.i32("options"); o.threads = r.i32("options"); o.seed = r.u32("options");
    get_geometry(r, o.dev);
    if (r.ok() && (o.particles < 1 || o.patch_size != 32 || !(o.resolution > 0) || o.dev.dir_dim < 8 || o.dev.max_beams < 1 || o.dev.pool_slots < 0))
        r.fail("bad options");
    const uint32_t P = r.ok() ? o.particles : 0;
    // front-end state
    const SE2 prior = r.se2("state"), odom = r.se2("state");
    const bool has_first = r.u8("state");
    const double acc_trans = r.f64("state"), acc_rot = r.f64("state"), neff = r.f64("state");
    std::vector<SE2> pose(r.count(P, 4 * 8, "poses"));
    for (SE2& p : pose) p = r.se2("poses");
    std::vector<double> weight, nweight, wsum;
    r.array(weight, P, "weights");
    r.array(nweight, P, "weights");
    r.array(wsum, P, "weights");
    std::vector<int32_t> last_idx;
    r.array(last_idx, r.u32("resample indices"), "resample indices");
    const uint64_t rs_count = r.u64("resample digest"), rs_hash = r.u64("resample digest"), scans_seen = r.u64("resample digest");
    std::vector<double> stamps;
    r.array(stamps, r.u32("timestamps"), "timestamps");
    const Counters last = get_counters(r), total = get_counters(r);
    const uint64_t detached_seen = r.u64("counters");
    double summary[4];
    for (double& v : summary) v = r.f64("summary");
    std::vector<Node> nodes(r.count(r.u32("nodes"), 4 * 8 + 4, "nodes"));
    for (size_t n = 0; n < nodes.size(); ++n) {
        nodes[n].pose   = r.se2("nodes");
        nodes[n].parent = r.i32("nodes");
        if (r.ok() && (nodes[n].parent < -1 || nodes[n].parent >= (int)n)) r.fail("a trajectory node does not follow its parent");
    }
    std::vector<int32_t> node_of;
    r.array(node_of, P, "trajectory heads");
    const std::string rng = r.str("random generator");
    if (r.ok()) {
        for (int32_t v : last_idx)
            if (v < 0 || v >= (int32_t)P) r.fail("resample index out of range");
        if (!last_idx.empty() && last_idx.size() != P) r.fail("resample indices of the wrong length");
        for (int32_t v : node_of)
            if (v < -1 || v >= (int32_t)nodes.size() || (has_first && v < 0)) r.fail("trajectory head out of range");
        if (!ckpt_check_rng(rng)) r.fail("malformed random generator state");
        if (!finite_se2(prior) || !finite_se2(odom)) r.fail("non-finite pose");
    }
    EngineImage img;
    bool present = false;
    if (r.ok()) ckpt_get_engine(r, &present, img, (int)P, 0);
    if (r.ok() && has_first && !present) r.fail("a filter past its first scan without device state");
    if (r.ok() && r.left() != 0) r.fail("bytes after the last section");
    if (!r.ok()) { err = r.error(); return nullptr; }
    if (!geometry_matches(dev, o.dev, present ? &img : nullptr, err)) return nullptr;
    s.encode_ms += ms_since(t1);
    // the file is valid: from here on the device
    if (cuda_device_count() < 1) { *code = LAMA_ERR_NO_DEVICE; err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    o.dev.device = dev.device; o.dev.stream = dev.stream; o.dev.timing = dev.timing;
    std::unique_ptr<PFSlam2D> p(create(o, err));
    if (!p) return nullptr;
    p->prior_ = prior; p->odom_ = odom; p->has_first_ = has_first;
    p->acc_trans_ = acc_trans; p->acc_rot_ = acc_rot; p->neff_ = neff;
    p->pose_ = pose; p->weight_ = weight; p->nweight_ = nweight; p->wsum_ = wsum;
    p->last_idx_ = last_idx;
    p->resample_count_ = rs_count; p->resample_hash_ = rs_hash; p->scans_seen_ = scans_seen;
    p->timestamps_ = stamps;
    p->last_ = last; p->total_ = total; p->detached_seen_ = detached_seen;
    p->t_sample_ = summary[0]; p->t_solve_ = summary[1]; p->t_norm_ = summary[2]; p->t_resample_ = summary[3];
    p->nodes_ = nodes; p->node_of_.assign(node_of.begin(), node_of.end());
    std::istringstream in(rng);
    in >> p->gen_;
    if (present) {
        Engine* e = Engine::restore(img, dev.device, dev.stream, err, &s.dev);
        if (!e) { *code = LAMA_ERR_CUDA; return nullptr; }
        p->eng_.reset(e);
        e->enable_timing(dev.timing != 0);
    }
    s.used_slots = img.used;
    s.references = sum_refs(img);
    s.total_ms   = ms_since(t0);
    *code = LAMA_OK;
    return p.release();
}

int Slam2D::save(const std::string& path, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    EngineImage img;
    if (eng_) {
        const int rc = eng_->snapshot(&img, &s.dev);
        if (rc != LAMA_OK) { err_ = eng_->last_error(); return rc; }
    }
    const auto t1 = clk::now();
    CkptWriter w;
    ckpt_put(w);
    ckpt_put_engine(w, eng_ ? &img : nullptr);
    s.encode_ms = ms_since(t1);
    std::string err;
    const int rc = ckpt_write_file(path, opt_.lidar_odometry ? kCkptLidarOdometry2D : kCkptSlam2D, w, {{img.slot_bytes, (size_t)img.used * img.slot_stride()}}, err, &s);
    if (rc != LAMA_OK) { err_ = err; return rc; }
    s.used_slots = img.used;
    s.references = sum_refs(img);
    s.total_ms   = ms_since(t0);
    return LAMA_OK;
}

Slam2D* Slam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    std::vector<uint8_t> file;
    uint32_t kind = 0;
    *code = ckpt_read_file(path, file, &kind, err, &s);
    if (*code != LAMA_OK) return nullptr;
    *code = LAMA_ERR_ARG;
    if (kind != kCkptSlam2D && kind != kCkptLidarOdometry2D) {
        err = wrong_kind(kind, "Slam2D");
        return nullptr;
    }
    const auto t1 = clk::now();
    CkptReader r(file.data() + kCkptHeaderBytes, file.size() - kCkptHeaderBytes);
    SlamSaved sv;
    ckpt_get(r, kind == kCkptLidarOdometry2D, sv);
    EngineImage img;
    bool present = false;
    if (r.ok()) ckpt_get_engine(r, &present, img, 1, sv.opt.occupancy == 1 ? 1 : 0);
    if (r.ok() && sv.has_first && !present) r.fail("a Slam2D past its first scan without device state");
    if (r.ok() && r.left() != 0) r.fail("bytes after the last section");
    if (!r.ok()) { err = r.error(); return nullptr; }
    if (!geometry_matches(dev, sv.opt.dev, present ? &img : nullptr, err)) return nullptr;
    s.encode_ms += ms_since(t1);
    if (cuda_device_count() < 1) { *code = LAMA_ERR_NO_DEVICE; err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    std::unique_ptr<Slam2D> p(ckpt_restore(sv, present ? &img : nullptr, dev, err, code, &s.dev));
    if (!p) return nullptr;
    s.used_slots = img.used;
    s.references = sum_refs(img);
    s.total_ms   = ms_since(t0);
    *code = LAMA_OK;
    return p.release();
}

void Slam2D::ckpt_put(CkptWriter& w) const
{
    for (double v : {opt_.trans_thresh, opt_.rot_thresh, opt_.l2_max, opt_.truncated_ray, opt_.truncated_range, opt_.resolution}) w.f64(v);
    w.u32(opt_.patch_size); w.u32(opt_.max_iter); w.i32(opt_.strategy); w.i32(opt_.occupancy);
    w.u8(opt_.transient_map); w.u8(opt_.lidar_odometry);
    put_geometry(w, opt_.dev);
    w.se2(pose_); w.se2(odom_); w.se2(map_update_pose_);
    w.u8(has_first_); w.u8(engine_ready_);
    w.u32(processed_); w.u64(removed_); w.u64(map_updates_);
    put_counters(w, last_); put_counters(w, total_);
}

void Slam2D::ckpt_get(CkptReader& r, bool lidar_odometry, SlamSaved& s)
{
    SlamOptions& o = s.opt;
    for (double* v : {&o.trans_thresh, &o.rot_thresh, &o.l2_max, &o.truncated_ray, &o.truncated_range, &o.resolution}) *v = r.f64("options");
    o.patch_size = r.u32("options"); o.max_iter = r.u32("options"); o.strategy = r.i32("options"); o.occupancy = r.i32("options");
    o.transient_map = r.u8("options"); o.lidar_odometry = r.u8("options");
    get_geometry(r, o.dev);
    if (r.ok() && (o.patch_size != 32 || !(o.resolution > 0) || o.occupancy < 0 || o.occupancy > 1 || o.dev.dir_dim < 8 || o.dev.max_beams < 1 ||
                   o.dev.pool_slots < 0 || o.lidar_odometry != lidar_odometry))
        r.fail("bad options");
    s.pose = r.se2("state"); s.odom = r.se2("state"); s.map_update_pose = r.se2("state");
    s.has_first = r.u8("state"); s.engine_ready = r.u8("state");
    s.processed = r.u32("state");
    s.removed = r.u64("state"); s.map_updates = r.u64("state");
    s.last = get_counters(r); s.total = get_counters(r);
    if (r.ok() && (!finite_se2(s.pose) || !finite_se2(s.odom) || !finite_se2(s.map_update_pose))) r.fail("non-finite pose");
}

Slam2D* Slam2D::ckpt_restore(const SlamSaved& s, const EngineImage* img, const DeviceOptions& dev, std::string& err, int* code, CheckpointTimes* t)
{
    SlamOptions o = s.opt;
    o.dev.device = dev.device; o.dev.stream = dev.stream; o.dev.timing = dev.timing;
    std::unique_ptr<Slam2D> p(create(o, err));
    if (!p) return nullptr;
    p->pose_ = s.pose; p->odom_ = s.odom; p->map_update_pose_ = s.map_update_pose;
    p->has_first_ = s.has_first; p->engine_ready_ = s.engine_ready;
    p->processed_ = s.processed; p->removed_ = s.removed; p->map_updates_ = s.map_updates;
    p->last_ = s.last; p->total_ = s.total;
    if (img) {
        Engine* e = Engine::restore(*img, dev.device, dev.stream, err, t);
        if (!e) { *code = LAMA_ERR_CUDA; return nullptr; }
        p->eng_.reset(e);
        e->enable_timing(dev.timing != 0);
        e->set_lidar_odometry_rays(o.lidar_odometry);
    }
    return p.release();
}

// ---- GraphSlam2D (kind 4) ---------------------------------------------------------------------------------------------------------------
namespace {
void put_loss(CkptWriter& w, const PgoLoss& l)
{
    for (double v : l.sigma) w.f64(v);
    w.f64(l.huber_k);
}
PgoLoss get_loss(CkptReader& r, const char* what)
{
    PgoLoss l;
    for (double& v : l.sigma) v = r.f64(what);
    l.huber_k = r.f64(what);
    bool ok = l.huber_k >= 0 && std::isfinite(l.huber_k);
    for (double v : l.sigma) ok = ok && v > 0 && std::isfinite(v);   // GraphSlam2D's sigmas are finite constants; inf would drop a factor
    if (r.ok() && !ok) r.fail(std::string("bad loss (") + what + ")");
    return l;
}
void put_betweens(CkptWriter& w, const std::vector<PgoBetween>& v)
{
    w.u32((uint32_t)v.size());
    for (const PgoBetween& b : v) {
        w.i32(b.from); w.i32(b.to); w.se2(b.measured);
        put_loss(w, b.loss);
    }
}
void get_betweens(CkptReader& r, std::vector<PgoBetween>& v, size_t n_keys, const char* what)
{
    v.resize(r.count(r.u32(what), 2 * 4 + 4 * 8 + 4 * 8, what));
    for (PgoBetween& b : v) {
        b.from = r.i32(what); b.to = r.i32(what); b.measured = r.se2(what);
        b.loss = get_loss(r, what);
        if (r.ok() && (b.from < 0 || (size_t)b.from >= n_keys || b.to < 0 || (size_t)b.to >= n_keys)) r.fail(std::string("a factor names no key (") + what + ")");
        if (r.ok() && !finite_se2(b.measured)) r.fail(std::string("non-finite factor (") + what + ")");
    }
}
bool finite3(const double* v, int n)
{
    for (int k = 0; k < n; ++k)
        if (!std::isfinite(v[k])) return false;
    return true;
}
}  // namespace

int GraphSlam2D::save(const std::string& path, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    Engine* ie = slam_->engine();
    const bool global = mapping_keyid_ > 0 && occ_;   // only then does the next generate_occupancy_map draw on occ_
    EngineImage inner, gimg;
    if (ie) {
        const int rc = ie->snapshot(&inner, &s.dev);
        if (rc != LAMA_OK) { err_ = ie->last_error(); return rc; }
    }
    if (global) {
        CheckpointTimes t;
        const int rc = occ_->engine()->snapshot(&gimg, &t);
        if (rc != LAMA_OK) { err_ = occ_->engine()->last_error(); return rc; }
        add_times(s.dev, t);
    }
    const auto t1 = clk::now();
    CkptWriter w;
    // graph options
    w.f64(opt_.key_pose_distance); w.f64(opt_.key_pose_angular_distance); w.i32(opt_.key_pose_head_delay);
    w.f64(opt_.loop_search_max_distance); w.f64(opt_.loop_search_min_distance); w.i32(opt_.loop_max_candidates);
    w.f64(opt_.loop_closure_scan_rmse); w.i32(opt_.loop_closure_max_candidates); w.i32(opt_.ignore_n_chain_poses);
    // the inner Slam2D: the bytes of a kind-2 file's options and state
    slam_->ckpt_put(w);
    // graph state
    w.se2(correction_); w.se2(prev_);
    w.f64(accdist_); w.f64(factordist_);
    w.u64(mapping_keyid_);
    w.u64(stats_.loop_factors); w.u64(stats_.optimizations); w.u64(stats_.optimizations_ok);
    const PgoReport& rep = stats_.last;
    w.i32(rep.status); w.u32(rep.iterations); w.u32(rep.lambda_tries); w.u64(rep.cg_iterations);
    w.f64(rep.initial_error); w.f64(rep.final_error); w.f64(rep.device_ms);
    w.u32((uint32_t)last_candidates_.size());
    for (int c : last_candidates_) w.i32(c);
    double c[2];
    slam_window_center(slam_.get(), c);   // a restored engine does not know its centre (Engine::set_center)
    w.f64(c[0]); w.f64(c[1]);
    // key poses
    w.u32((uint32_t)keys_.size());
    for (const KeyPose& k : keys_) {
        w.i32(k.id); w.se2(k.pose); w.se2(k.original);
        for (double v : k.origin) w.f64(v);
        for (double v : k.quat) w.f64(v);
        w.f64(k.stamp);
        w.u32((uint32_t)(k.pts.size() / 3));
        w.bytes(k.pts.data(), k.pts.size() * 8);
    }
    w.u32((uint32_t)links_.size());
    for (const auto& l : links_) { w.i32(l.first); w.i32(l.second); }
    // the pose graph
    w.u32((uint32_t)priors_.size());
    for (const PgoPrior& p : priors_) {
        w.i32(p.node); w.se2(p.measured);
        put_loss(w, p.loss);
    }
    put_betweens(w, factors_);
    put_betweens(w, queue_);
    // the inner engine, its slots, the global map's engine and its slots
    ckpt_put_engine(w, ie ? &inner : nullptr);
    CkptWriter g;
    g.buf.clear();
    ckpt_put_engine(g, global ? &gimg : nullptr);
    s.encode_ms = ms_since(t1);
    std::string err;
    const int rc = ckpt_write_file(path, kCkptGraphSlam2D, w,
                                   {{inner.slot_bytes, (size_t)inner.used * inner.slot_stride()}, {g.buf.data(), g.buf.size()},
                                    {gimg.slot_bytes, (size_t)gimg.used * gimg.slot_stride()}},
                                   err, &s);
    if (rc != LAMA_OK) { err_ = err; return rc; }
    s.used_slots = (uint64_t)inner.used + gimg.used;
    s.references = sum_refs(inner) + sum_refs(gimg);
    s.total_ms   = ms_since(t0);
    return LAMA_OK;
}

GraphSlam2D* GraphSlam2D::load(const std::string& path, const DeviceOptions& dev, std::string& err, int* code, CheckpointStats* st)
{
    const auto t0 = clk::now();
    CheckpointStats local;
    CheckpointStats& s = st ? *st : local;
    s = CheckpointStats();
    std::vector<uint8_t> file;
    uint32_t kind = 0;
    *code = ckpt_read_file(path, file, &kind, err, &s);
    if (*code != LAMA_OK) return nullptr;
    *code = LAMA_ERR_ARG;
    if (kind != kCkptGraphSlam2D) {
        err = wrong_kind(kind, "GraphSlam2D");
        return nullptr;
    }
    const auto t1 = clk::now();
    CkptReader r(file.data() + kCkptHeaderBytes, file.size() - kCkptHeaderBytes);
    GraphOptions g;
    g.key_pose_distance = r.f64("graph options"); g.key_pose_angular_distance = r.f64("graph options"); g.key_pose_head_delay = r.i32("graph options");
    g.loop_search_max_distance = r.f64("graph options"); g.loop_search_min_distance = r.f64("graph options"); g.loop_max_candidates = r.i32("graph options");
    g.loop_closure_scan_rmse = r.f64("graph options"); g.loop_closure_max_candidates = r.i32("graph options"); g.ignore_n_chain_poses = r.i32("graph options");
    // an infinite threshold is a user's way to switch a test off (key_pose_angular_distance = inf: keys by distance only), so only NaN is refused
    bool nan = false;
    for (double v : {g.key_pose_distance, g.key_pose_angular_distance, g.loop_search_max_distance, g.loop_search_min_distance, g.loop_closure_scan_rmse})
        nan = nan || std::isnan(v);
    if (r.ok() && (nan || g.key_pose_head_delay < 0 || g.ignore_n_chain_poses < 0 || g.loop_max_candidates < 0)) r.fail("bad graph options");
    SlamSaved sv;
    Slam2D::ckpt_get(r, false, sv);
    if (r.ok() && (!sv.opt.transient_map || sv.opt.truncated_ray != 1.0 || sv.opt.occupancy != 0))
        r.fail("the inner Slam2D's options are not the ones GraphSlam2D forces (transient map, truncated_ray 1, frequency map, no lidar odometry)");
    // graph state
    const SE2 correction = r.se2("graph state"), prev = r.se2("graph state");
    const double accdist = r.f64("graph state"), factordist = r.f64("graph state");
    const uint64_t mapping_keyid = r.u64("graph state");
    Stats stats;
    stats.loop_factors = r.u64("graph stats"); stats.optimizations = r.u64("graph stats"); stats.optimizations_ok = r.u64("graph stats");
    stats.last.status = r.i32("last report"); stats.last.iterations = r.u32("last report"); stats.last.lambda_tries = r.u32("last report");
    stats.last.cg_iterations = r.u64("last report");
    stats.last.initial_error = r.f64("last report"); stats.last.final_error = r.f64("last report"); stats.last.device_ms = r.f64("last report");
    std::vector<int32_t> cands;
    r.array(cands, r.u32("last candidates"), "last candidates");
    double center[2];
    center[0] = r.f64("window centre"); center[1] = r.f64("window centre");
    if (r.ok() && (!finite_se2(correction) || !finite_se2(prev) || !std::isfinite(accdist) || !std::isfinite(factordist) || !finite3(center, 2)))
        r.fail("non-finite graph state");
    // key poses: every one at least 136 bytes before its points
    std::vector<KeyPose> keys(r.count(r.u32("key poses"), 4 + 2 * 32 + 7 * 8 + 8 + 4, "key poses"));
    for (size_t i = 0; i < keys.size() && r.ok(); ++i) {
        KeyPose& k = keys[i];
        k.id = r.i32("key pose"); k.pose = r.se2("key pose"); k.original = r.se2("key pose");
        for (double& v : k.origin) v = r.f64("key pose");
        for (double& v : k.quat) v = r.f64("key pose");
        k.stamp = r.f64("key pose");
        const size_t m = r.count(r.u32("key points"), 24, "key points");
        r.array(k.pts, 3 * m, "key points");
        if (r.ok() && k.id != (int)i) r.fail("a key pose id differs from its index");
        if (r.ok() && (!finite_se2(k.pose) || !finite_se2(k.original) || !finite3(k.origin, 3) || !finite3(k.quat, 4))) r.fail("non-finite key pose");
    }
    const size_t n = keys.size();
    auto is_key = [n](int32_t v) { return v >= 0 && (size_t)v < n; };
    std::vector<int32_t> link_ids;
    r.array(link_ids, 2 * (uint64_t)r.count(r.u32("links"), 8, "links"), "links");
    std::vector<PgoPrior> priors(r.count(r.u32("priors"), 4 + 4 * 8 + 4 * 8, "priors"));
    for (PgoPrior& p : priors) {
        p.node = r.i32("priors"); p.measured = r.se2("priors");
        p.loss = get_loss(r, "priors");
        if (r.ok() && !is_key(p.node)) r.fail("a prior names no key");
        if (r.ok() && !finite_se2(p.measured)) r.fail("non-finite prior");
    }
    std::vector<PgoBetween> factors, queue;
    get_betweens(r, factors, n, "factors");
    get_betweens(r, queue, n, "loop-factor queue");
    if (r.ok()) {
        for (int32_t v : link_ids)
            if (!is_key(v)) r.fail("a link names no key");
        for (int32_t v : cands)
            if (!is_key(v)) r.fail("a loop candidate names no key");
        if (mapping_keyid > n) r.fail("mapping key id past the key poses");
    }
    EngineImage inner, gimg;
    bool inner_present = false, global_present = false;
    if (r.ok()) ckpt_get_engine(r, &inner_present, inner, 1, 0, false);
    if (r.ok() && inner_present && inner.known_plane) r.fail("the inner engine has a known plane");
    if (r.ok() && (sv.has_first || n > 0) && !inner_present) r.fail("a GraphSlam2D past its first scan without device state");
    if (r.ok()) ckpt_get_engine(r, &global_present, gimg, 1, 0, true);
    if (r.ok() && global_present && !gimg.known_plane) r.fail("the global map's engine has no known plane");
    if (r.ok() && global_present != (mapping_keyid > 0)) r.fail("a global map section must be present exactly when the mapping key id is above 0");
    if (r.ok() && r.left() != 0) r.fail("bytes after the last section");
    if (!r.ok()) { err = r.error(); return nullptr; }
    if (!geometry_matches(dev, sv.opt.dev, inner_present ? &inner : nullptr, err)) return nullptr;
    s.encode_ms += ms_since(t1);
    // the file is valid: from here on the device
    if (cuda_device_count() < 1) { *code = LAMA_ERR_NO_DEVICE; err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    std::unique_ptr<Slam2D> slam(Slam2D::ckpt_restore(sv, inner_present ? &inner : nullptr, dev, err, code, &s.dev));
    if (!slam) return nullptr;
    if (slam->engine()) slam->engine()->set_center(center[0], center[1]);
    std::unique_ptr<GraphSlam2D> p(new GraphSlam2D());
    g.slam = sv.opt;
    g.slam.dev.device = dev.device; g.slam.dev.stream = dev.stream; g.slam.dev.timing = dev.timing;   // pgo_optimize_graph runs there
    p->opt_ = g;
    p->slam_ = std::move(slam);
    if (global_present) {
        CheckpointTimes t;
        Engine* e = Engine::restore(gimg, dev.device, dev.stream, err, &t);
        if (!e) { *code = LAMA_ERR_CUDA; return nullptr; }
        e->enable_timing(dev.timing != 0);
        p->occ_.reset(OccupancyMapDev::adopt(e));
        add_times(s.dev, t);
    }
    p->mapping_keyid_ = (size_t)mapping_keyid;
    p->keys_ = std::move(keys);
    for (size_t i = 0; i < link_ids.size(); i += 2) p->links_.push_back({link_ids[i], link_ids[i + 1]});
    p->priors_ = std::move(priors);
    p->factors_ = std::move(factors);
    p->queue_ = std::move(queue);
    p->last_candidates_.assign(cands.begin(), cands.end());
    p->correction_ = correction;
    p->accdist_ = accdist;
    p->prev_ = prev;
    p->factordist_ = factordist;
    p->stats_ = stats;
    s.used_slots = (uint64_t)inner.used + gimg.used;
    s.references = sum_refs(inner) + sum_refs(gimg);
    s.total_ms   = ms_since(t0);
    *code = LAMA_OK;
    return p.release();
}

}  // namespace lama_b200
