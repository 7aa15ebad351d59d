// frontend.cpp -- host orchestration of PFSlam2D / Slam2D / Loc2D over the device Engine.
#include "frontend.h"
#include "render_plan.h"
#include "rng_skip.h"
#include "sdm_io.h"
#include "window_guard.h"

#include <cuda_runtime.h>

#include "shard_comm.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>
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

// Before an update of `count` particles at predicted poses `poses`: moves the engine's window so that every cell the update can touch
// lies inside it (window_guard.h), or leaves it where it is when no window holds that box.  `grow` (m) widens the box on every side.
static int follow_window(Engine* e, const SE2* poses, int count, const double* origin, const double* quat, const double* pts, int n, double grow = 0.0)
{
    const EngineConfig& c = e->config();
    const uint32_t reach = (uint32_t)std::lround(std::sqrt((double)e->max_sqdist()));
    double mn[2], mx[2];
    guard_box(poses, count, moving_tf(origin, quat), pts, n, c.resolution, reach, mn, mx);
    for (int k = 0; k < 2; ++k) {
        mn[k] -= grow;
        mx[k] += grow;
    }
    const double robot[2] = {poses[0].tx, poses[0].ty};
    int32_t base[2];
    if (window_guard(e->window(), mn, mx, robot, 1.0 / c.resolution, base) != kGuardShift) return LAMA_OK;
    return e->shift_window(base[0], base[1]);
}

// =====================================================================================================
// PFSlam2D
// =====================================================================================================
bool PFSlam2D::valid_options(const PFOptions& o, std::string& err)
{
    if (o.particles < 1) { err = "PFSlam2D: Options::particles must be set (>= 1)"; return false; }
    if (o.patch_size != 32) { err = "PFSlam2D: only patch_size 32 is supported on the device"; return false; }
    { uint32_t r; if (!Engine::reach_fits(o.resolution, o.l2_max, &r, err)) { err = "PFSlam2D: " + err; return false; } }
    if (o.shard_count < 1 || o.shard_rank >= o.shard_count || o.particles % o.shard_count != 0) {
        err = "PFSlam2D: particles must divide evenly over shard_count";
        return false;
    }
    if (o.shard_count > 1 && o.seed == 0) {
        // seed 0 means "take one from random_device" (pf_slam2d.cpp:131-132): every rank would draw its own, the ranks' odometry
        // noise and resampling indices would differ and the map migration would pair up the wrong particles
        err = "PFSlam2D: sharded operation needs an explicit (non-zero) seed shared by all ranks (with seed 0 each rank draws its own)";
        return false;
    }
    return true;
}

void PFSlam2D::place()
{
    P_ = opt_.particles;
    const int per = (int)(opt_.particles / opt_.shard_count);
    lo_ = (int)opt_.shard_rank * per;
    hi_ = lo_ + per;
    if (opt_.seed == 0) opt_.seed = std::random_device{}();  // pf_slam2d.cpp:131-132
}

PFSlam2D* PFSlam2D::create(const PFOptions& o, std::string& err)
{
    if (!valid_options(o, err)) return nullptr;
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    PFSlam2D* p = new PFSlam2D();
    p->opt_ = o;
    p->place();
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
    if (comm_) shard_comm_destroy(comm_);
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

// Start of a pipelined scan.  `moved` false = motion gate (pf_slam2d.cpp:215-222): the previous scan's counters are booked and nothing else
// happens for this scan.  Otherwise the previous scan's counters go to *prev (*prev_pending: its map update is still to be collected)
// and a staged scan is selected (*staged: the step uploads no scan).
int PFSlam2D::begin_step(const double* origin, const double* quat, bool moved, bool* did_update, Counters* prev, bool* prev_pending, bool* staged)
{
    if (!moved) {
        int rcs = settle_counters();
        last_ = Counters();
        last_idx_.clear();
        staged_index_ = -1;
        return rcs;
    }
    *did_update = true;
    *prev = last_;
    *prev_pending = counters_pending_;
    counters_pending_ = false;
    last_ = Counters();
    last_idx_.clear();
    const int index = staged_index_;
    staged_index_ = -1;
    *staged = index >= 0;
    if (*staged) {
        int rc = eng_->select_staged(index, origin, quat, opt_.truncated_ray, opt_.truncated_range);
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    return LAMA_OK;
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
    Counters prev;
    bool prev_pending = false, staged = false;
    int rc = begin_step(origin, quat, moved, did_update, &prev, &prev_pending, &staged);
    if (rc != LAMA_OK || !moved) return rc;
    const int nl = hi_ - lo_;
    std::vector<HostMatchResult> res((size_t)nl);
    rc = eng_->step_async(staged ? nullptr : pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range, &pose_[lo_], nl,
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
    if (moved) {
        const bool staged = staged_index_ >= 0;
        int rcw = follow_window(eng_.get(), &pose_[lo_], hi_ - lo_, origin, quat, staged ? staged_host_.data() + (size_t)staged_index_ * staged_beams_ * 3 : pts,
                                staged ? staged_beams_ : n);
        if (rcw != LAMA_OK) return engine_fail(rcw);
    }
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
    bool ok = d_send_.alloc(payload) == cudaSuccess && d_recv_.alloc(payload * opt_.shard_count) == cudaSuccess &&
              h_recv_.alloc(payload * opt_.shard_count) == cudaSuccess && d_tab_.alloc((size_t)P_ * 3 * 2) == cudaSuccess &&
              h_tab_.alloc((size_t)P_ * 3 * 2) == cudaSuccess;
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
    Counters prev;
    bool prev_pending = false, staged = false;
    int rc = begin_step(origin, quat, moved, did_update, &prev, &prev_pending, &staged);
    if (rc != LAMA_OK || !moved) return rc;
    const int nl = hi_ - lo_, G = (int)opt_.shard_count;
    rc = eng_->step_enqueue(staged ? nullptr : pts, n, origin, quat, opt_.truncated_ray, opt_.truncated_range, &pose_[lo_], nl, make_solver(0, opt_.max_iter),
                            opt_.meas_sigma);
    if (rc != LAMA_OK) return engine_fail(rc);
    const size_t payload = (size_t)nl * kShardF + 1;
    rc = eng_->pack_results(nl, digest_, d_send_.get(), shard_stream(comm_));   // waits for the match on the communicator's stream
    if (rc != LAMA_OK) return engine_fail(rc);
    if (shard_allgather(comm_, d_send_.get(), d_recv_.get(), payload * 8) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
    if (cudaMemcpyAsync(h_recv_.get(), d_recv_.get(), payload * 8 * G, cudaMemcpyDeviceToHost, (cudaStream_t)shard_stream(comm_)) != cudaSuccess)
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
        const double* src = h_recv_.get() + (size_t)r * payload;
        if (src[(size_t)nl * kShardF] != h_recv_.get()[(size_t)nl * kShardF]) return fail("the resampling decision diverged between ranks", LAMA_ERR_STATE);
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
    std::memcpy(h_tab_.get(), mine.data(), mine.size() * 8);
    int64_t* d_all = d_tab_.get() + (size_t)P_ * 3;
    int64_t* h_all = h_tab_.get() + (size_t)P_ * 3;
    if (cudaMemcpyAsync(d_tab_.get(), h_tab_.get(), mine.size() * 8, cudaMemcpyHostToDevice, cs) != cudaSuccess) return fail("migrate: size table upload failed", LAMA_ERR_CUDA);
    if (shard_allgather(comm_, d_tab_.get(), d_all, mine.size() * 8) != 0) return fail(shard_error(comm_), LAMA_ERR_CUDA);
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
    const double* scan_pts = staged_index_ >= 0 ? staged_host_.data() + (size_t)staged_index_ * staged_beams_ * 3 : pts;
    const int scan_n = staged_index_ >= 0 ? staged_beams_ : n;
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
    if (opt_.shard_count == 1) {   // sharded ranks keep a fixed window
        rc = follow_window(eng_.get(), &pose_[lo_], hi_ - lo_, origin, quat, scan_pts, scan_n);
        if (rc != LAMA_OK) return engine_fail(rc);
    }
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
        if (rc != LAMA_OK) return engine_fail(rc);
    }
    return LAMA_OK;
}

int PFSlam2D::stage_scans(const double* pts, int n_scans, int n)
{
    if (!pts || n_scans < 1 || n < 1) return fail("stage_scans: bad arguments", LAMA_ERR_ARG);
    staged_scans_ = n_scans;
    staged_beams_ = n;
    staged_host_.assign(pts, pts + (size_t)n_scans * n * 3);   // the window guard reads the points of every update on the host
    if (eng_) {
        int rc = eng_->stage_scans(pts, n_scans, n);
        return rc == LAMA_OK ? rc : engine_fail(rc);
    }
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

void Slam2D::window_center(double c[2])
{
    if (eng_) {
        c[0] = eng_->config().center_x;
        c[1] = eng_->config().center_y;
    } else {
        c[0] = pose_.tx;
        c[1] = pose_.ty;
    }
}

int GraphSlam2D::generate_occupancy_map(bool full, OccupancyMapDev** out)
{
    if (mapping_keyid_ == 0 || !occ_) {   // :132-133
        double c[2];
        slam_->window_center(c);
        const double res = full ? opt_.slam.resolution : 0.1;
        // a rebuild after an optimisation casts every key again: start at the pool the previous map of this resolution grew to
        const int start = occ_ && occ_->engine()->config().resolution == res ? occ_->engine()->config().pool_slots : 0;
        OccupancyMapDev* m = OccupancyMapDev::create(res, 32, c[0], c[1], slam_->device_options(), err_, start);
        if (!m) return LAMA_ERR_CUDA;
        m->set_follow(true);
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
    slam_->window_center(c);
    {   // centred where the inner map's window now is: the creation centre moved by the patches between the window the engine was
        // created with around it and the window it has now
        const EngineConfig& ec = e->config();
        const double scale = 1.0 / ec.resolution, patch = (double)kPatchLen * ec.resolution;
        const DirWindow w = e->window();
        c[0] += (double)(w.base_px - ((int32_t)(w2m(c[0], scale) >> kPatchLog2) - w.dim / 2)) * patch;
        c[1] += (double)(w.base_py - ((int32_t)(w2m(c[1], scale) >> kPatchLog2) - w.dim / 2)) * patch;
    }
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
bool Slam2D::valid_options(const SlamOptions& o, std::string& err)
{
    if (o.patch_size != 32) { err = "Slam2D: only patch_size 32 is supported on the device"; return false; }
    { uint32_t r; if (!Engine::reach_fits(o.resolution, o.l2_max, &r, err)) { err = "Slam2D: " + err; return false; } }
    return true;
}

Slam2D* Slam2D::create(const SlamOptions& o, std::string& err)
{
    if (!valid_options(o, err)) return nullptr;
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
    if (rc == LAMA_OK) rc = follow_window(eng_.get(), &pose_, 1, origin, quat, pts, n);
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
        if (rc == LAMA_OK) rc = follow_window(eng_.get(), &pose_, 1, origin, quat, pts, n);
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
    if (rc == LAMA_OK) rc = follow_window(eng_.get(), &pose_, 1, origin, quat, pts, n);
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
    d->growable_ = dev.pool_slots <= 0;
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

OccupancyMapDev* OccupancyMapDev::create(double resolution, uint32_t patch_size, double cx, double cy, const DeviceOptions& dev, std::string& err,
                                         int start_slots)
{
    if (patch_size != 32) { err = "FrequencyOccupancyMap: only patch_size 32 is supported on the device"; return nullptr; }
    if (cuda_device_count() < 1) { err = "no CUDA device available: the lama_b200 hot path has no CPU fallback"; return nullptr; }
    EngineConfig cfg = engine_config(dev, 1, resolution, resolution, cx, cy);   // no distance map is kept: the smallest reach
    const bool growable = cfg.pool_slots <= 0;
    if (growable) cfg.pool_slots = std::max(cfg.dir_dim * cfg.dir_dim, (int)std::min<int64_t>(start_slots, kPoolSlotCap));
    cfg.known_plane = true;
    Engine* en = Engine::create(cfg, err);
    if (!en) return nullptr;
    OccupancyMapDev* m = new OccupancyMapDev();
    m->eng_.reset(en);
    m->growable_ = growable;
    en->enable_timing(dev.timing != 0);
    return m;
}

OccupancyMapDev* OccupancyMapDev::adopt(Engine* e, bool growable)
{
    OccupancyMapDev* m = new OccupancyMapDev();
    m->eng_.reset(e);
    m->growable_ = growable;
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
    const uint64_t key = m2p(x, y);
    auto it = patches_.find(key);
    if (it == patches_.end()) it = patches_.emplace(key, std::vector<int8_t>(kPatchCells, 0)).first;
    it->second[cell_index(x, y)] = (int8_t)(state < 0 ? -1 : (state > 0 ? 1 : 0));
}
bool SimpleOccupancyHost::is_free_world(double wx, double wy) const
{
    const uint32_t x = w2m(wx, scale_), y = w2m(wy, scale_);
    auto it = patches_.find(m2p(x, y));
    return it != patches_.end() && it->second[cell_index(x, y)] == -1;
}
bool SimpleOccupancyHost::bounds_world(double mn[2], double mx[2]) const
{
    if (patches_.empty()) return false;
    uint32_t lo[2] = {0xffffffffu, 0xffffffffu}, hi[2] = {0, 0};
    for (auto& kv : patches_) {
        uint32_t ax, ay;
        p2m(kv.first, ax, ay);
        lo[0] = std::min(lo[0], ax); lo[1] = std::min(lo[1], ay);
        hi[0] = std::max(hi[0], ax); hi[1] = std::max(hi[1], ay);
    }
    for (int k = 0; k < 2; ++k) {
        mn[k] = ((double)lo[k] - (double)kMapOffsetCells) / scale_;               // Map::m2w
        mx[k] = ((double)(hi[k] + kPatchLen) - (double)kMapOffsetCells) / scale_;
    }
    return true;
}

// ---- per-robot steps of Loc2D ---------------------------------------------------------------------------------------
std::vector<double> loc_sampling_steps(double resolution)
{
    std::vector<double> st;
    const double sstep = resolution;   // loc2d.cpp:93-107
    auto add = [&](double x, double y) { st.push_back(x); st.push_back(y); };
    add(0.0, 0.0);
    for (int i = 1; i <= 20; ++i) {
        add(i * sstep, 0.0); add(0.0, i * sstep); add(-i * sstep, 0.0); add(0.0, -i * sstep);
        add(i * sstep, i * sstep); add(-i * sstep, i * sstep); add(i * sstep, -i * sstep); add(-i * sstep, -i * sstep);
    }
    return st;
}

bool loc_predict(LocRobot& r, const LocOptions& o, const SE2& odometry, bool force)
{
    const SE2 odelta = se2_mul(se2_inv(r.odom), odometry);
    const SE2 ppose  = se2_mul(r.pose, odelta);
    const bool enough = !(xy_norm(odelta) <= o.trans_thresh && std::abs(se2_rotation(odelta)) <= o.rot_thresh);
    if (!force && !enough) return false;
    r.pose = ppose;
    r.odom = odometry;
    return true;
}

bool loc_gloc_step(LocRobot& r, const LocOptions& o)
{
    if (!r.do_gloc) return false;
    if (r.gloc_cur_iter < o.gloc_iters) {
        r.gloc_cur_iter++;
        return true;
    }
    r.do_gloc       = false;
    r.gloc_cur_iter = 0;
    return false;
}

bool loc_gloc_candidates(LocRobot& r, const LocOptions& o, const SimpleOccupancyHost& occ, std::vector<SE2>& cand)
{
    double mn[2], mx[2];
    if (!occ.bounds_world(mn, mx)) return false;
    const double diff[2] = {mx[0] - mn[0], mx[1] - mn[1]};
    cand.resize(o.gloc_particles);
    auto uniform = [&]() { std::uniform_real_distribution<double> d(0.0, 1.0); return d(r.gen); };
    for (uint32_t i = 0; i < o.gloc_particles; ++i) {
        double x, y, a;
        for (;;) {
            x = mn[0] + uniform() * diff[0];
            y = mn[1] + uniform() * diff[1];
            if (!occ.is_free_world(x, y)) continue;
            a = uniform() * 2 * M_PI - M_PI;
            break;
        }
        cand[i] = se2_from_xyr(x, y, a);
    }
    return true;
}

void loc_gloc_winner(LocRobot& r, const SE2* cand, const HostMatchResult* res, size_t n)
{
    double best = std::numeric_limits<double>::max();
    for (size_t i = 0; i < n; ++i)
        if (res[i].sums[10] < best) {  // residuals.squaredNorm()
            best   = res[i].sums[10];
            r.pose = cand[i];
        }
}

void loc_tracked(LocRobot& r, const HostMatchResult& res, size_t n)
{
    r.pose  = res.state;
    r.iters = res.iterations;
    r.evals = res.evals_ref + 2;  // + the covariance and rmse evaluations of solver.cpp:110 / loc2d.cpp:178
    covariance_from_sums(res.sums, n, r.cov);
}

void loc_sampling_blend(LocRobot& r, const std::vector<double>& steps, const double* l, double alpha)
{
    const int n_off = (int)(steps.size() / 2);
    double K[4] = {0, 0, 0, 0}, u[2] = {0, 0}, sl = 0;
    for (int i = 0; i < n_off; ++i) {
        const double x = r.pose.tx + steps[2 * i], y = r.pose.ty + steps[2 * i + 1];
        K[0] = K[0] + x * x * l[i]; K[1] = K[1] + x * y * l[i]; K[2] = K[2] + y * x * l[i]; K[3] = K[3] + y * y * l[i];
        u[0] = u[0] + x * l[i]; u[1] = u[1] + y * l[i];
        sl = sl + l[i];
    }
    const double a = 1.0 / sl, b = 1.0 / (sl * sl);
    const double sc[4] = {a * K[0] - b * u[0] * u[0], a * K[1] - b * u[0] * u[1], a * K[2] - b * u[1] * u[0], a * K[3] - b * u[1] * u[1]};
    double* cov = r.cov;
    cov[0] = alpha * sc[0] + (1.0 - alpha) * cov[0]; cov[1] = alpha * sc[1] + (1.0 - alpha) * cov[1];
    cov[3] = alpha * sc[2] + (1.0 - alpha) * cov[3]; cov[4] = alpha * sc[3] + (1.0 - alpha) * cov[4];
}

void loc_finish(LocRobot& r, const LocOptions& o, const HostMatchResult& res, size_t n)
{
    r.rmse = std::sqrt(res.sums[10] / ((double)(n - 1)));  // loc2d.cpp:178-180
    if (r.do_gloc && r.rmse < o.gloc_thresh) {             // loc2d.cpp:182-188
        r.do_gloc       = false;
        r.gloc_cur_iter = 0;
    }
}

// ---- Loc2D -----------------------------------------------------------------------------------------------------------
Loc2D* Loc2D::create(const LocOptions& o, std::string& err)
{
    DistanceMapDev* dm = DistanceMapDev::create(o.resolution, o.patch_size, o.l2_max, o.center_x, o.center_y, o.dev, err);
    if (!dm) return nullptr;
    Loc2D* l = new Loc2D();
    l->opt_ = o;
    l->dm_.reset(dm);
    l->occ_.reset(new SimpleOccupancyHost(o.resolution));
    l->cov_blend_ = std::max(std::min(o.cov_blend, 1.0), 0.0);  // loc2d.cpp:90
    l->sampling_steps_ = loc_sampling_steps(o.resolution);
    return l;
}

// Loc2D::globalLocalization (loc2d.cpp:249-286): candidates are drawn on the host with the reference's rejection
// sampling (same generator calls in the same order), evaluated in ONE device launch (the same evaluation kernel as
// scan matching, every block on the same map) and the best is chosen with the reference's strict `<` in index order.
// The candidates cover the whole SimpleOccupancyMap, which has no window.  When the distance map follows and has parked patches the
// launch is k_match_extent, which reads every patch (Engine::match_extent).  With nothing parked every patch is in the window, and
// k_match reads a cell outside it as absent, as the reference's const get does.
int Loc2D::global_localization(int n)
{
    std::vector<SE2> cand;
    if (!loc_gloc_candidates(rb_, opt_, *occ_, cand)) return LAMA_OK;
    std::vector<HostMatchResult> res(cand.size());
    SolverOptions so = make_solver(0, 0);
    Engine* eng = dm_->engine();
    int rc = eng->follows() && eng->has_parked() ? eng->match_extent(cand.data(), (int)cand.size(), so, 0.05, res.data())
                                                 : eng->match(cand.data(), (int)cand.size(), 0, true, so, 0.05, 1, res.data());
    if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
    loc_gloc_winner(rb_, cand.data(), res.data(), cand.size());
    (void)n;
    return LAMA_OK;
}

// A Loc2D follows exactly when its distance map does: before a device read at the pose, the window moves over the guarded box of the
// scan at the pose (window_guard.h), grown by the reach of the sampling covariance's offsets (20 steps of one resolution,
// loc_sampling_steps).  On a static map a shift only moves directory entries to and from the parked lists.
int Loc2D::follow(const double* pts, int n, const double* origin, const double* quat)
{
    Engine* eng = dm_->engine();
    if (!eng->follows()) return LAMA_OK;
    const int rc = follow_window(eng, &rb_.pose, 1, origin, quat, pts, n, 20.0 * opt_.resolution);
    if (rc != LAMA_OK) err_ = eng->last_error();
    return rc;
}

// Loc2D::addSamplingCovariance (loc2d.cpp:199-247)
int Loc2D::add_sampling_covariance(const double* pts, int n, const double* origin, const double* quat)
{
    const int n_off = (int)(sampling_steps_.size() / 2);
    const int stride = (int)std::max((size_t)n / 100, (size_t)1);
    std::vector<double> l((size_t)n_off);
    int rc = follow(pts, n, origin, quat);
    if (rc == LAMA_OK) rc = dm_->engine()->sampling_likelihood(0, rb_.pose, sampling_steps_.data(), n_off, stride, l.data());
    if (rc != LAMA_OK) { err_ = dm_->engine()->last_error(); return rc; }
    loc_sampling_blend(rb_, sampling_steps_, l.data(), cov_blend_);
    return LAMA_OK;
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
    if (!rb_.has_first) {  // loc2d.cpp:128-141
        rb_.odom      = odometry;
        rb_.has_first = true;
        if (!force) { *did_update = true; return LAMA_OK; }
        rc = eng->set_scan(pts, n, origin, quat, 0, 0);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
        scan_set = true;
        HostMatchResult r;
        rc = follow(pts, n, origin, quat);
        if (rc == LAMA_OK) rc = eng->match(&rb_.pose, 1, 0, false, so, 0.05, 1, &r);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
        rb_.rmse = std::sqrt(r.sums[10] / ((double)((size_t)n - 1)));
    }
    if (!loc_predict(rb_, opt_, odometry, force)) return LAMA_OK;
    if (!scan_set) {
        rc = eng->set_scan(pts, n, origin, quat, 0, 0);
        if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
    }
    if (loc_gloc_step(rb_, opt_)) {  // loc2d.cpp:154-166
        rc = global_localization(n);
        if (rc != LAMA_OK) return rc;
    }
    HostMatchResult r;
    rc = follow(pts, n, origin, quat);
    if (rc == LAMA_OK) rc = eng->match(&rb_.pose, 1, 0, false, so, 0.05, 0, &r);
    if (rc != LAMA_OK) { err_ = eng->last_error(); return rc; }
    loc_tracked(rb_, r, (size_t)n);
    if (cov_blend_ > 0.0) {     // loc2d.cpp:175-176
        rc = add_sampling_covariance(pts, n, origin, quat);
        if (rc != LAMA_OK) return rc;
    }
    loc_finish(rb_, opt_, r, (size_t)n);
    *did_update = true;
    return LAMA_OK;
}

// ---- Loc2DFleet ------------------------------------------------------------------------------------------------------
Loc2DFleet* Loc2DFleet::create(const LocOptions& o, int robots, std::string& err)
{
    if (robots < 1) { err = "a fleet needs at least one robot"; return nullptr; }
    DistanceMapDev* dm = DistanceMapDev::create(o.resolution, o.patch_size, o.l2_max, o.center_x, o.center_y, o.dev, err);
    if (!dm) return nullptr;
    std::unique_ptr<Loc2DFleet> f(new Loc2DFleet());
    f->opt_ = o;
    f->dm_.reset(dm);
    f->occ_.reset(new SimpleOccupancyHost(o.resolution));
    f->cov_blend_ = std::max(std::min(o.cov_blend, 1.0), 0.0);
    f->sampling_steps_ = loc_sampling_steps(o.resolution);
    f->rb_.resize((size_t)robots);
    if (dm->engine()->fleet_reserve(robots, f->sampling_steps_.data(), (int)(f->sampling_steps_.size() / 2)) != LAMA_OK) {
        err = dm->engine()->last_error();
        return nullptr;
    }
    return f.release();
}

int Loc2DFleet::fail(int rc)
{
    err_ = dm_->engine()->last_error();
    return rc;
}

// One round.  The stand-alone first forced update also evaluates the RMSE at the pose before the prediction (loc2d.cpp:134-140); the
// same update overwrites it after the tracking match, so the round leaves that evaluation out.
int Loc2DFleet::update(int count, const int* robots, const double* pts, const int* n_points, const double* origins, const double* quats, const double* odom_xyr,
                       const int* force, int* did_update)
{
    const int R = (int)rb_.size();
    const int max_beams = dm_->engine()->config().max_beams;
    if (count < 1 || count > R || !robots || !pts || !n_points || !odom_xyr || !did_update) { err_ = "null argument or count out of range"; return LAMA_ERR_ARG; }
    std::vector<uint8_t> seen((size_t)R, 0);
    for (int k = 0; k < count; ++k) {
        if (robots[k] < 0 || robots[k] >= R) { err_ = "robot " + std::to_string(robots[k]) + " out of range"; return LAMA_ERR_ARG; }
        if (seen[(size_t)robots[k]]++) { err_ = "robot " + std::to_string(robots[k]) + " appears twice in one update"; return LAMA_ERR_ARG; }
        if (n_points[k] < 1 || n_points[k] > max_beams) { err_ = "scan " + std::to_string(k) + ": number of points out of range [1, max_beams]"; return LAMA_ERR_ARG; }
    }
    for (int k = 0; k < count; ++k) did_update[k] = 0;
    int rc = dm_->flush_if_pending();
    if (rc != LAMA_OK) { err_ = dm_->error(); return rc; }
    Engine* eng = dm_->engine();

    // the robots that go on (loc2d.cpp:128-152), their scans in call order
    std::vector<int> go;                 // call index
    std::vector<size_t> first(count);    // first point of scan k
    size_t np = 0;
    for (int k = 0; k < count; ++k) { first[k] = np; np += (size_t)n_points[k]; }
    for (int k = 0; k < count; ++k) {
        LocRobot& r = rb_[(size_t)robots[k]];
        const double* od = odom_xyr + 3 * (size_t)k;
        const SE2 odometry = se2_from_xyr(od[0], od[1], od[2]);
        const bool f = force && force[k];
        if (!r.has_first) {
            r.odom      = odometry;
            r.has_first = true;
            if (!f) { did_update[k] = 1; continue; }
        }
        if (loc_predict(r, opt_, odometry, f)) go.push_back(k);
    }
    if (go.empty()) return LAMA_OK;
    const int G = (int)go.size();
    {
        std::vector<double> p;
        std::vector<int> n(G);
        std::vector<double> o, q;
        for (int j = 0; j < G; ++j) {
            const int k = go[j];
            p.insert(p.end(), pts + 3 * first[k], pts + 3 * (first[k] + n_points[k]));
            n[j] = n_points[k];
            if (origins) o.insert(o.end(), origins + 3 * k, origins + 3 * k + 3);
            if (quats) q.insert(q.end(), quats + 4 * k, quats + 4 * k + 4);
        }
        rc = eng->fleet_scans(p.data(), n.data(), G, origins ? o.data() : nullptr, quats ? q.data() : nullptr);
        if (rc != LAMA_OK) return fail(rc);
    }

    // global localisation of every robot that runs it this round: one launch over all candidates, winners on the host
    {
        std::vector<SE2> cand, c;
        std::vector<int32_t> blocks;
        std::vector<std::pair<int, size_t>> owners;   // (go index, first candidate)
        for (int j = 0; j < G; ++j) {
            LocRobot& r = rb_[(size_t)robots[go[j]]];
            if (!loc_gloc_step(r, opt_) || !loc_gloc_candidates(r, opt_, *occ_, c)) continue;
            owners.emplace_back(j, cand.size());
            cand.insert(cand.end(), c.begin(), c.end());
            blocks.insert(blocks.end(), c.size(), j);
        }
        if (!cand.empty()) {
            std::vector<HostMatchResult> res(cand.size());
            rc = eng->match_fleet(blocks.data(), cand.data(), (int)cand.size(), 1, make_solver(0, 0), 0.05);
            if (rc == LAMA_OK) rc = eng->fleet_results(res.data(), nullptr);
            if (rc != LAMA_OK) return fail(rc);
            for (const auto& ow : owners)
                loc_gloc_winner(rb_[(size_t)robots[go[ow.first]]], cand.data() + ow.second, res.data() + ow.second, opt_.gloc_particles);
        }
    }

    // tracking of every robot that goes on, then the sampling likelihoods at the solved poses: one read-back
    std::vector<SE2> poses(G);
    std::vector<int32_t> blocks(G);
    for (int j = 0; j < G; ++j) { poses[j] = rb_[(size_t)robots[go[j]]].pose; blocks[j] = j; }
    std::vector<HostMatchResult> res(G);
    const size_t n_off = sampling_steps_.size() / 2;
    std::vector<double> lik(cov_blend_ > 0.0 ? (size_t)G * n_off : 0);
    rc = eng->match_fleet(blocks.data(), poses.data(), G, 0, make_solver(opt_.strategy, opt_.max_iter), 0.05);
    if (rc == LAMA_OK && cov_blend_ > 0.0) rc = eng->sampling_fleet();
    if (rc == LAMA_OK) rc = eng->fleet_results(res.data(), lik.data());
    if (rc != LAMA_OK) return fail(rc);
    for (int j = 0; j < G; ++j) {
        const int k = go[j];
        LocRobot& r = rb_[(size_t)robots[k]];
        loc_tracked(r, res[j], (size_t)n_points[k]);
        if (cov_blend_ > 0.0) loc_sampling_blend(r, sampling_steps_, lik.data() + (size_t)j * n_off, cov_blend_);
        loc_finish(r, opt_, res[j], (size_t)n_points[k]);
        did_update[k] = 1;
    }
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

}  // namespace lama_b200
