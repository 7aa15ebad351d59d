// oracle_capi.cpp -- flat C entry points over lama_oracle.hpp for the ctypes test harness.
// TEST INFRASTRUCTURE ONLY (see the header of lama_oracle.hpp).  Built by oracle/Makefile into
// oracle/_build/liblama_oracle.so; loaded only by tests/, __graft_entry__.smoke() and the
// cpu_baseline / --impl reference legs of bench.py.
#include "lama_oracle.hpp"

using namespace orc;

namespace {
PointCloud make_cloud(const double* pts, int n, const double* origin, const double* quat)
{
    PointCloud pc;
    pc.pts.assign(pts, pts + 3 * (size_t)n);
    if (origin) for (int i = 0; i < 3; ++i) pc.origin[i] = origin[i];
    if (quat) for (int i = 0; i < 4; ++i) pc.quat[i] = quat[i];
    return pc;
}
SE2 se2_from(const double* s) { return SE2(SO2{s[0], s[1]}, s[2], s[3]); }
void se2_to(const SE2& s, double* o) { o[0] = s.r.c; o[1] = s.r.s; o[2] = s.tx; o[3] = s.ty; }

template <typename M, typename F>
void export_window(const M& map, uint32_t x0, uint32_t y0, int w, int h, F&& f)
{
    for (int j = 0; j < h; ++j)
        for (int i = 0; i < w; ++i) {
            Vec3u c{x0 + (uint32_t)i, y0 + (uint32_t)j, (uint32_t)map.offset};
            auto it = map.patches.find(map.m2p(c));
            if (it == map.patches.end()) { f(j * w + i, nullptr, false); continue; }
            uint32_t ci = map.m2c(c);
            f(j * w + i, &it->second->cells[ci], it->second->is_on(ci));
        }
}
template <typename M>
int map_bounds(const M& map, uint32_t* mn, uint32_t* mx)
{
    if (map.patches.empty()) return 0;
    mn[0] = mn[1] = 0xffffffffu;
    mx[0] = mx[1] = 0;
    for (auto& kv : map.patches) {
        Vec3u a = map.p2m(kv.first);
        mn[0] = std::min(mn[0], a.x); mn[1] = std::min(mn[1], a.y);
        mx[0] = std::max(mx[0], a.x); mx[1] = std::max(mx[1], a.y);
    }
    mx[0] += map.patch_length; mx[1] += map.patch_length;
    return (int)map.patches.size();
}
void export_dm(const DynamicDistanceMap& dm, uint32_t x0, uint32_t y0, int w, int h, uint16_t* sqdist, uint8_t* valid,
               uint8_t* known, int16_t* ox, int16_t* oy, uint8_t* queued)
{
    export_window(dm, x0, y0, w, h, [&](int k, const DistCell* c, bool on) {
        if (sqdist) sqdist[k] = c ? c->sqdist : 0;
        if (valid) valid[k] = c ? c->valid_obstacle : 0;
        if (known) known[k] = on;
        if (ox) ox[k] = c ? c->ox : 0;
        if (oy) oy[k] = c ? c->oy : 0;
        if (queued) queued[k] = c ? c->is_queued : 0;
    });
}
void export_occ(const FrequencyOccupancyMap& occ, uint32_t x0, uint32_t y0, int w, int h, uint16_t* occupied, uint16_t* visited, uint8_t* known)
{
    export_window(occ, x0, y0, w, h, [&](int k, const FreqCell* c, bool on) {
        if (occupied) occupied[k] = c ? c->occupied : 0;
        if (visited) visited[k] = c ? c->visited : 0;
        if (known) known[k] = on;
    });
}
}  // namespace

// OccupancyMap::{getProbability, isFree, isOccupied, isUnknown}(Vector3ui) for n cells; flags bit 0 free, 1 occupied, 2 unknown
template <class M>
static void occ_query(const M& m, const uint32_t* cells, int n, double* prob, uint8_t* flags)
{
    for (int i = 0; i < n; ++i) {
        const Vec3u c{cells[2 * i], cells[2 * i + 1], 0};
        prob[i]  = m.get_probability(c);
        flags[i] = (uint8_t)((m.is_free(c) ? 1 : 0) | (m.is_occupied(c) ? 2 : 0) | (m.is_unknown(c) ? 4 : 0));
    }
}

extern "C" {

// ---- Lie / pose algebra ----------------------------------------------------------------------
void orc_se2_from_xyr(double x, double y, double r, double* out) { se2_to(SE2(r, x, y), out); }
void orc_se2_exp(const double* h, double* out) { se2_to(SE2::exp(h), out); }
void orc_se2_mul(const double* a, const double* b, double* out) { se2_to(se2_from(a) * se2_from(b), out); }
void orc_se2_inv(const double* a, double* out) { se2_to(se2_from(a).inverse(), out); }
double orc_se2_log_rot(const double* a) { return se2_from(a).r.log(); }

// ---- RNG -------------------------------------------------------------------------------------
void* orc_rng_create(uint32_t seed) { auto* r = new Random; r->seed(seed); return r; }
void orc_rng_destroy(void* r) { delete (Random*)r; }
double orc_rng_uniform(void* r) { return ((Random*)r)->uniform(); }
double orc_rng_normal(void* r, double sigma) { return ((Random*)r)->normal(sigma); }
uint32_t orc_rng_raw(void* r) { return ((Random*)r)->gen(); }

// ---- grid addressing / ray ------------------------------------------------------------------------
void orc_w2m(double res, uint32_t patch, const double* p, uint32_t* out)
{
    SparseMap<FreqCell> m(res, patch);
    Vec3u c = m.w2m(p);
    out[0] = c.x; out[1] = c.y; out[2] = c.z;
}
void orc_w2m_nocast(double res, uint32_t patch, const double* p, double* out) { SparseMap<FreqCell>(res, patch).w2m_nocast(p, out); }
uint64_t orc_m2p(double res, uint32_t patch, const uint32_t* c) { return SparseMap<FreqCell>(res, patch).m2p(Vec3u{c[0], c[1], c[2]}); }
uint32_t orc_m2c(double res, uint32_t patch, const uint32_t* c) { return SparseMap<FreqCell>(res, patch).m2c(Vec3u{c[0], c[1], c[2]}); }
int orc_ray(const uint32_t* from, const uint32_t* to, uint32_t* out, int cap)
{
    int n = 0;
    SparseMap<FreqCell>::compute_ray(Vec3u{from[0], from[1], from[2]}, Vec3u{to[0], to[1], to[2]}, [&](const Vec3u& c) {
        if (n < cap) { out[3 * n] = c.x; out[3 * n + 1] = c.y; out[3 * n + 2] = c.z; }
        ++n;
    });
    return n;
}

// ---- stand-alone DDM --------------------------------------------------------------------------------
void* orc_ddm_create(double res, uint32_t patch, double l2_max)
{
    auto* d = new DynamicDistanceMap(res, patch);
    d->set_max_distance(l2_max);
    return d;
}
void* orc_ddm_clone(void* d) { return new DynamicDistanceMap(*(DynamicDistanceMap*)d); }
void orc_ddm_destroy(void* d) { delete (DynamicDistanceMap*)d; }
void orc_ddm_set_shuffle(void* d, uint32_t s) { ((DynamicDistanceMap*)d)->set_shuffle(s); }
uint64_t orc_ddm_peak_queue(void* d) { return ((DynamicDistanceMap*)d)->peak_queue; }
uint32_t orc_ddm_max_sqdist(void* d) { return ((DynamicDistanceMap*)d)->max_sqdist_; }
void orc_ddm_add(void* d, const uint32_t* cells, int n)
{
    for (int i = 0; i < n; ++i) ((DynamicDistanceMap*)d)->add_obstacle(Vec3u{cells[2 * i], cells[2 * i + 1], (uint32_t)((DynamicDistanceMap*)d)->offset});
}
void orc_ddm_remove(void* d, const uint32_t* cells, int n)
{
    for (int i = 0; i < n; ++i) ((DynamicDistanceMap*)d)->remove_obstacle(Vec3u{cells[2 * i], cells[2 * i + 1], (uint32_t)((DynamicDistanceMap*)d)->offset});
}
uint32_t orc_ddm_update(void* d) { return ((DynamicDistanceMap*)d)->update(); }
void orc_ddm_distance(void* d, const double* pts, int n, double* dist, double* grad)
{
    auto* dm = (DynamicDistanceMap*)d;
    for (int i = 0; i < n; ++i) dist[i] = dm->distance(&pts[3 * i], grad ? &grad[3 * i] : nullptr);
}
void orc_ddm_distance_cells(void* d, const uint32_t* cells, int n, double* dist)
{
    auto* dm = (DynamicDistanceMap*)d;
    for (int i = 0; i < n; ++i) dist[i] = dm->distance(Vec3u{cells[2 * i], cells[2 * i + 1], (uint32_t)dm->offset});
}
int orc_ddm_bounds(void* d, uint32_t* mn, uint32_t* mx) { return map_bounds(*(DynamicDistanceMap*)d, mn, mx); }
void orc_ddm_export(void* d, uint32_t x0, uint32_t y0, int w, int h, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                    int16_t* oy, uint8_t* queued)
{
    export_dm(*(DynamicDistanceMap*)d, x0, y0, w, h, sqdist, valid, known, ox, oy, queued);
}

// ---- scan matching on a DDM -----------------------------------------------------------------------------
void orc_match_eval(void* d, const double* pts, int n, const double* origin, const double* quat, const double* state, double* r, double* J)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    MatchSurface2D ms((DynamicDistanceMap*)d, &pc, se2_from(state));
    std::vector<double> rr, jj;
    ms.eval(rr, J ? &jj : nullptr);
    std::copy(rr.begin(), rr.end(), r);
    if (J) std::copy(jj.begin(), jj.end(), J);
}
// weighted normal equations at `state`: out = {A00,A01,A02,A11,A12,A22, g0,g1,g2, chi2, sum_d2}
void orc_match_normal_eq(void* d, const double* pts, int n, const double* origin, const double* quat, const double* state, int robust_kind,
                         double robust_param, double* out)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    MatchSurface2D ms((DynamicDistanceMap*)d, &pc, se2_from(state));
    std::vector<double> r, J;
    ms.eval(r, &J);
    RobustCost rc;
    rc.kind  = (RobustCost::Kind)robust_kind;
    rc.param = robust_param;
    double sd2 = 0;
    for (size_t i = 0; i < r.size(); ++i) {
        sd2 += r[i] * r[i];
        double w = std::sqrt(rc.value(r[i]));
        r[i] *= w; J[3 * i] *= w; J[3 * i + 1] *= w; J[3 * i + 2] *= w;
    }
    double g[3], A[9], chi2;
    Strategy::normal_eq(r, J, g, A, chi2);
    out[0] = A[0]; out[1] = A[1]; out[2] = A[2]; out[3] = A[4]; out[4] = A[5]; out[5] = A[8];
    out[6] = g[0]; out[7] = g[1]; out[8] = g[2]; out[9] = chi2; out[10] = sd2;
}
// the 3x3 solve of one GN / LM step: A h = b, A row-major 3 x 3 (lower triangle referenced)
void orc_ldlt_solve3(const double* A, const double* b, double* h) { ldlt_solve3(A, b, h); }
// full solve; state in/out; stats = {iterations, evals}
void orc_match_solve(void* d, const double* pts, int n, const double* origin, const double* quat, double* state, int strategy, int robust_kind,
                     double robust_param, uint32_t max_iter, double* cov, uint32_t* stats)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    MatchSurface2D ms((DynamicDistanceMap*)d, &pc, se2_from(state));
    SolverOptions so;
    so.max_iterations = max_iter;
    so.strategy.kind  = (Strategy::Kind)strategy;
    so.robust.kind    = (RobustCost::Kind)robust_kind;
    so.robust.param   = robust_param;
    SolveStats st     = solve(so, ms, cov);
    se2_to(ms.state, state);
    if (stats) { stats[0] = st.iterations; stats[1] = st.evals; }
}

// ---- GraphSlam2D loop-closure front end -------------------------------------------------------------------
int orc_loop_closure_candidates(const double* key_xy, int n_keys, int ignore_n, const double* query, double radius, int max_candidates, int* ids)
{
    std::vector<double> k(key_xy, key_xy + 2 * (size_t)n_keys);
    std::vector<int> v = find_loop_closure_candidates(k, ignore_n, query, radius, (size_t)max_candidates);
    for (size_t i = 0; i < v.size(); ++i) ids[i] = v[i];
    return (int)v.size();
}
double orc_match_error(void* d, const double* pts, int n, const double* origin, const double* quat, const double* state)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return match_error(*(DynamicDistanceMap*)d, pc, se2_from(state));
}
double orc_correlate_candidate_scan(void* d, const double* pts, int n, const double* origin, const double* quat, const double* ref_xyr, const double* cand_xyr,
                                    double* between_xyr)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    Pose2D between;
    double rmse = correlate_candidate_scan(*(DynamicDistanceMap*)d, pc, Pose2D(ref_xyr[0], ref_xyr[1], ref_xyr[2]), Pose2D(cand_xyr[0], cand_xyr[1], cand_xyr[2]), between);
    between_xyr[0] = between.x(); between_xyr[1] = between.y(); between_xyr[2] = between.rotation();
    return rmse;
}
double orc_coarse_correlate_candidate_scan(void* d, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat, const double* pts, int n,
                                           const double* origin, const double* quat, const double* ref_xyr, const double* cand_xyr, double* between_xyr)
{
    PointCloud rc = make_cloud(ref_pts, ref_n, ref_origin, ref_quat), pc = make_cloud(pts, n, origin, quat);
    Pose2D between;
    double rmse = coarse_correlate_candidate_scan(*(DynamicDistanceMap*)d, rc, pc, Pose2D(ref_xyr[0], ref_xyr[1], ref_xyr[2]), Pose2D(cand_xyr[0], cand_xyr[1], cand_xyr[2]),
                                                  between);
    between_xyr[0] = between.x(); between_xyr[1] = between.y(); between_xyr[2] = between.rotation();
    return rmse;
}

// ---- PFSlam2D --------------------------------------------------------------------------------------------
struct orc_pf_options {
    uint32_t particles;
    double srr, str, stt, srt, meas_sigma, meas_sigma_gain, trans_thresh, rot_thresh, l2_max, truncated_ray, truncated_range, resolution;
    uint32_t patch_size, max_iter;
    int32_t threads;
    uint32_t seed;
};
void* orc_pf_create(const orc_pf_options* o)
{
    PFOptions p;
    p.particles = o->particles; p.srr = o->srr; p.str = o->str; p.stt = o->stt; p.srt = o->srt;
    p.meas_sigma = o->meas_sigma; p.meas_sigma_gain = o->meas_sigma_gain; p.trans_thresh = o->trans_thresh; p.rot_thresh = o->rot_thresh;
    p.l2_max = o->l2_max; p.truncated_ray = o->truncated_ray; p.truncated_range = o->truncated_range; p.resolution = o->resolution;
    p.patch_size = o->patch_size; p.max_iter = o->max_iter; p.threads = o->threads; p.seed = o->seed;
    return new PFSlam2D(p);
}
void orc_pf_destroy(void* h) { delete (PFSlam2D*)h; }
void orc_pf_set_prior(void* h, double x, double y, double r) { ((PFSlam2D*)h)->set_prior(Pose2D(x, y, r)); }
// bench only: change the size of the thread pool of a running filter (the reference fixes it in the constructor, pf_slam2d.cpp:123-128)
void orc_pf_set_threads(void* h, int32_t n)
{
    auto* pf = (PFSlam2D*)h;
    pf->opt.threads = n;
    pf->pool.reset(n > 1 ? new ThreadPool((size_t)n) : nullptr);
}
void orc_pf_set_shuffle(void* h, uint32_t s) { ((PFSlam2D*)h)->shuffle_ties = s; }
int orc_pf_update(void* h, const double* pts, int n, const double* origin, const double* quat, const double* odom_xyr)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return ((PFSlam2D*)h)->update(pc, Pose2D(odom_xyr[0], odom_xyr[1], odom_xyr[2])) ? 1 : 0;
}
double orc_pf_neff(void* h) { return ((PFSlam2D*)h)->neff; }
int orc_pf_best(void* h) { return (int)((PFSlam2D*)h)->best_particle_idx(); }
// states: P x 4 (c,s,tx,ty); weights: P x 3 (weight, normalized_weight, weight_sum)
void orc_pf_get_particles(void* h, double* states, double* weights)
{
    auto* pf = (PFSlam2D*)h;
    auto& ps = pf->particles[pf->cur];
    for (size_t i = 0; i < ps.size(); ++i) {
        if (states) se2_to(ps[i].pose.state, &states[4 * i]);
        if (weights) { weights[3 * i] = ps[i].weight; weights[3 * i + 1] = ps[i].normalized_weight; weights[3 * i + 2] = ps[i].weight_sum; }
    }
}
int orc_pf_last_resample(void* h, int32_t* idx)
{
    auto* pf = (PFSlam2D*)h;
    for (size_t i = 0; i < pf->last_sample_idx.size(); ++i) idx[i] = pf->last_sample_idx[i];
    return (int)pf->last_sample_idx.size();
}
// counters: {evals, ray_cells, dm_pops, detached, gn_iters, resampled} for the last update and totals
void orc_pf_counters(void* h, uint64_t* last, uint64_t* total)
{
    auto* pf = (PFSlam2D*)h;
    const ScanCounters* src[2] = {&pf->last, &pf->total};
    uint64_t* dst[2] = {last, total};
    for (int k = 0; k < 2; ++k) {
        if (!dst[k]) continue;
        dst[k][0] = src[k]->evals; dst[k][1] = src[k]->ray_cells; dst[k][2] = src[k]->dm_pops;
        dst[k][3] = src[k]->detached; dst[k][4] = src[k]->gn_iters; dst[k][5] = (uint64_t)src[k]->resampled;
    }
}
void orc_pf_times(void* h, double* t) { auto* pf = (PFSlam2D*)h; t[0] = pf->t_solve; t[1] = pf->t_norm; t[2] = pf->t_resample; t[3] = pf->t_map; }
int orc_pf_trajectory(void* h, int particle, double* xyr, int cap)
{
    auto* pf = (PFSlam2D*)h;
    auto& poses = pf->particles[pf->cur][particle].poses;
    int n = (int)poses.size();
    for (int i = 0; i < n && i < cap; ++i) { xyr[3 * i] = poses[i].x(); xyr[3 * i + 1] = poses[i].y(); xyr[3 * i + 2] = poses[i].rotation(); }
    return n;
}
int orc_pf_dm_bounds(void* h, int particle, uint32_t* mn, uint32_t* mx) { auto* pf = (PFSlam2D*)h; return map_bounds(*pf->particles[pf->cur][particle].dm, mn, mx); }
int orc_pf_occ_bounds(void* h, int particle, uint32_t* mn, uint32_t* mx) { auto* pf = (PFSlam2D*)h; return map_bounds(*pf->particles[pf->cur][particle].occ, mn, mx); }
void orc_pf_export_dm(void* h, int particle, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                      int16_t* oy, uint8_t* queued)
{
    auto* pf = (PFSlam2D*)h;
    export_dm(*pf->particles[pf->cur][particle].dm, x0, y0, w, hh, sqdist, valid, known, ox, oy, queued);
}
void orc_pf_export_occ(void* h, int particle, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* occupied, uint16_t* visited, uint8_t* known)
{
    auto* pf = (PFSlam2D*)h;
    export_occ(*pf->particles[pf->cur][particle].occ, x0, y0, w, hh, occupied, visited, known);
}
void* orc_pf_dm_handle(void* h, int particle) { auto* pf = (PFSlam2D*)h; return pf->particles[pf->cur][particle].dm.get(); }

// ---- Slam2D ----------------------------------------------------------------------------------------------
struct orc_slam_options {
    double trans_thresh, rot_thresh, l2_max, truncated_ray, truncated_range, resolution;
    uint32_t patch_size, max_iter;
    int32_t strategy;
    int32_t transient_map;
};
void* orc_slam_create(const orc_slam_options* o)
{
    SlamOptions s;
    s.trans_thresh = o->trans_thresh; s.rot_thresh = o->rot_thresh; s.l2_max = o->l2_max; s.truncated_ray = o->truncated_ray;
    s.truncated_range = o->truncated_range; s.resolution = o->resolution; s.patch_size = o->patch_size; s.max_iter = o->max_iter;
    s.strategy = o->strategy; s.transient_map = o->transient_map != 0;
    return new Slam2D(s);
}
void orc_slam_destroy(void* h) { delete (Slam2D*)h; }
void orc_slam_set_pose(void* h, double x, double y, double r) { ((Slam2D*)h)->pose = Pose2D(x, y, r); }
void orc_slam_set_shuffle(void* h, uint32_t s) { ((Slam2D*)h)->dm.set_shuffle(s); }
// ---- Slam2D over the probabilistic (log-odds) occupancy map -------------------------------------------------------
void* orc_slamp_create(const orc_slam_options* o)
{
    SlamOptions s;
    s.trans_thresh = o->trans_thresh; s.rot_thresh = o->rot_thresh; s.l2_max = o->l2_max; s.truncated_ray = o->truncated_ray;
    s.truncated_range = o->truncated_range; s.resolution = o->resolution; s.patch_size = o->patch_size; s.max_iter = o->max_iter;
    s.strategy = o->strategy; s.transient_map = o->transient_map != 0;
    return new Slam2DProb(s);
}
void orc_slamp_destroy(void* h) { delete (Slam2DProb*)h; }
void orc_slamp_set_pose(void* h, double x, double y, double r) { ((Slam2DProb*)h)->pose = Pose2D(x, y, r); }
int orc_slamp_update(void* h, const double* pts, int n, const double* origin, const double* quat, const double* odom_xyr)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return ((Slam2DProb*)h)->update(pc, Pose2D(odom_xyr[0], odom_xyr[1], odom_xyr[2])) ? 1 : 0;
}
void orc_slamp_get_state(void* h, double* state) { se2_to(((Slam2DProb*)h)->pose.state, state); }
void orc_slamp_counters(void* h, uint64_t* last)
{
    auto* s = (Slam2DProb*)h;
    last[0] = s->last.evals; last[1] = s->last.ray_cells; last[2] = s->last.dm_pops; last[3] = 0; last[4] = s->last.gn_iters; last[5] = 0;
}
int orc_slamp_dm_bounds(void* h, uint32_t* mn, uint32_t* mx) { return map_bounds(((Slam2DProb*)h)->dm, mn, mx); }
int orc_slamp_occ_bounds(void* h, uint32_t* mn, uint32_t* mx) { return map_bounds(((Slam2DProb*)h)->occ, mn, mx); }
void orc_slamp_export_dm(void* h, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy,
                         uint8_t* queued)
{
    export_dm(((Slam2DProb*)h)->dm, x0, y0, w, hh, sqdist, valid, known, ox, oy, queued);
}
void orc_slamp_export_occ(void* h, uint32_t x0, uint32_t y0, int w, int hh, float* prob, uint8_t* known)
{
    export_window(((Slam2DProb*)h)->occ, x0, y0, w, hh, [&](int k, const ProbCell* c, bool on) {
        prob[k]  = c ? c->prob : 0.0f;
        known[k] = on;
    });
}
// applies a sequence of setOccupied (1) / setFree (0) calls to ONE cell of a fresh ProbabilisticOccupancyMap;
// prob_out[i] = cell value after call i, changed_out[i] = the call's return value
void orc_prob_sequence(const uint8_t* kinds, int n, float* prob_out, uint8_t* changed_out)
{
    ProbabilisticOccupancyMap m(0.05, 32);
    Vec3u c{(uint32_t)m.offset + 3, (uint32_t)m.offset + 5, (uint32_t)m.offset};
    for (int i = 0; i < n; ++i) {
        changed_out[i] = kinds[i] ? m.set_occupied(c) : m.set_free(c);
        prob_out[i]    = static_cast<const SparseMap<ProbCell>&>(m).get(c)->prob;
    }
}
// the constants of ProbabilisticOccupancyMap's constructor: {miss, hit, clamp_min, clamp_max, occ_thresh}
void orc_prob_constants(double* out)
{
    ProbabilisticOccupancyMap m(0.05, 32);
    out[0] = m.miss_; out[1] = m.hit_; out[2] = m.clamp_min_; out[3] = m.clamp_max_; out[4] = m.occ_thresh_;
}

int orc_slam_update(void* h, const double* pts, int n, const double* origin, const double* quat, const double* odom_xyr)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return ((Slam2D*)h)->update(pc, Pose2D(odom_xyr[0], odom_xyr[1], odom_xyr[2])) ? 1 : 0;
}
void orc_slam_get_state(void* h, double* state) { se2_to(((Slam2D*)h)->pose.state, state); }
void orc_slam_counters(void* h, uint64_t* last, uint64_t* total)
{
    auto* s = (Slam2D*)h;
    const ScanCounters* src[2] = {&s->last, &s->total};
    uint64_t* dst[2] = {last, total};
    for (int k = 0; k < 2; ++k) {
        if (!dst[k]) continue;
        dst[k][0] = src[k]->evals; dst[k][1] = src[k]->ray_cells; dst[k][2] = src[k]->dm_pops;
        dst[k][3] = src[k]->detached; dst[k][4] = src[k]->gn_iters; dst[k][5] = 0;
    }
}
int orc_slam_dm_bounds(void* h, uint32_t* mn, uint32_t* mx) { return map_bounds(((Slam2D*)h)->dm, mn, mx); }
int orc_slam_occ_bounds(void* h, uint32_t* mn, uint32_t* mx) { return map_bounds(((Slam2D*)h)->occ, mn, mx); }
void orc_slam_export_dm(void* h, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy,
                        uint8_t* queued)
{
    export_dm(((Slam2D*)h)->dm, x0, y0, w, hh, sqdist, valid, known, ox, oy, queued);
}
void orc_slam_export_occ(void* h, uint32_t x0, uint32_t y0, int w, int hh, uint16_t* occupied, uint16_t* visited, uint8_t* known)
{
    export_occ(((Slam2D*)h)->occ, x0, y0, w, hh, occupied, visited, known);
}
void* orc_slam_dm_handle(void* h) { return &((Slam2D*)h)->dm; }

// ---- Loc2D -------------------------------------------------------------------------------------------------
struct orc_loc_options {
    double trans_thresh, rot_thresh, l2_max, resolution;
    uint32_t patch_size, max_iter;
    int32_t strategy;
    uint32_t gloc_particles, gloc_iters;
    double gloc_thresh, cov_blend;
};
void* orc_loc_create(const orc_loc_options* o)
{
    LocOptions l;
    l.trans_thresh = o->trans_thresh; l.rot_thresh = o->rot_thresh; l.l2_max = o->l2_max; l.resolution = o->resolution;
    l.patch_size = o->patch_size; l.max_iter = o->max_iter; l.strategy = o->strategy;
    l.gloc_particles = o->gloc_particles; l.gloc_iters = o->gloc_iters; l.gloc_thresh = o->gloc_thresh; l.cov_blend = o->cov_blend;
    return new Loc2D(l);
}
void orc_loc_destroy(void* h) { delete (Loc2D*)h; }
void* orc_loc_dm_handle(void* h) { return &((Loc2D*)h)->dm; }
void orc_loc_set_seed(void* h, uint32_t seed) { ((Loc2D*)h)->rng.seed(seed); }
void orc_loc_trigger_gloc(void* h) { ((Loc2D*)h)->trigger_global_localization(); }
int orc_loc_gloc_active(void* h) { return ((Loc2D*)h)->do_global_localization ? 1 : 0; }
// SimpleOccupancyMap::setFree (-1) / setUnknown (0) / setOccupied (1) on n cells
void orc_loc_occ_set(void* h, const uint32_t* cells, int n, int state)
{
    auto* l = (Loc2D*)h;
    for (int i = 0; i < n; ++i) {
        Vec3u c{cells[2 * i], cells[2 * i + 1], (uint32_t)l->occ.offset};
        if (state < 0) l->occ.set_free(c);
        else if (state > 0) l->occ.set_occupied(c);
        else l->occ.set_unknown(c);
    }
}
void orc_loc_set_pose(void* h, double x, double y, double r) { ((Loc2D*)h)->set_pose(Pose2D(x, y, r)); }
int orc_loc_update(void* h, const double* pts, int n, const double* origin, const double* quat, const double* odom_xyr, int force)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return ((Loc2D*)h)->update(pc, Pose2D(odom_xyr[0], odom_xyr[1], odom_xyr[2]), force != 0) ? 1 : 0;
}
void orc_loc_get(void* h, double* state, double* cov, double* rmse, uint32_t* stats)
{
    auto* l = (Loc2D*)h;
    if (state) se2_to(l->pose.state, state);
    if (cov) std::copy(l->cov, l->cov + 9, cov);
    if (rmse) *rmse = l->rmse;
    if (stats) { stats[0] = l->last_stats.iterations; stats[1] = l->last_stats.evals; }
}


// ---- SDM persistence and image export (Map::write/read, sdm::export_to_png content) on map handles -------------------
void* orc_pf_occ_handle(void* h, int particle) { auto* pf = (PFSlam2D*)h; return pf->particles[pf->cur][particle].occ.get(); }
void* orc_slam_occ_handle(void* h) { return &((Slam2D*)h)->occ; }
void* orc_slamp_occ_handle(void* h) { return &((Slam2DProb*)h)->occ; }
void* orc_slamp_dm_handle(void* h) { return &((Slam2DProb*)h)->dm; }
void* orc_loc_occ_handle(void* h) { return &((Loc2D*)h)->occ; }
int orc_ddm_write(void* d, const char* path) { auto* m = (DynamicDistanceMap*)d; return m->write(path, &m->max_sqdist_, sizeof(m->max_sqdist_)) ? 1 : 0; }
int orc_ddm_read(void* d, const char* path) { auto* m = (DynamicDistanceMap*)d; return m->read(path, &m->max_sqdist_, sizeof(m->max_sqdist_)) ? 1 : 0; }
int orc_freq_write(void* d, const char* path) { return ((FrequencyOccupancyMap*)d)->write(path, nullptr, 0) ? 1 : 0; }
int orc_prob_write(void* d, const char* path) { return ((ProbabilisticOccupancyMap*)d)->write(path, nullptr, 0) ? 1 : 0; }
int orc_simple_write(void* d, const char* path) { return ((SimpleOccupancyMap*)d)->write(path, nullptr, 0) ? 1 : 0; }
int orc_simple_read(void* d, const char* path) { return ((SimpleOccupancyMap*)d)->read(path, nullptr, 0) ? 1 : 0; }
static int image_out(const std::vector<uint8_t>& img, uint32_t w, uint32_t h, uint8_t* out, size_t cap, int* dims)
{
    dims[0] = (int)w; dims[1] = (int)h;
    if (out && cap >= img.size()) std::memcpy(out, img.data(), img.size());
    return 1;
}
int orc_ddm_image(void* d, uint8_t* out, size_t cap, int* dims) { uint32_t w, h; auto img = distance_image(*(DynamicDistanceMap*)d, w, h); return image_out(img, w, h, out, cap, dims); }
int orc_freq_image(void* d, uint8_t* out, size_t cap, int* dims) { uint32_t w, h; auto img = occupancy_image(*(FrequencyOccupancyMap*)d, w, h); return image_out(img, w, h, out, cap, dims); }
int orc_prob_image(void* d, uint8_t* out, size_t cap, int* dims) { uint32_t w, h; auto img = occupancy_image(*(ProbabilisticOccupancyMap*)d, w, h); return image_out(img, w, h, out, cap, dims); }


// ---- LidarOdometry2D ------------------------------------------------------------------------------------------------
void* orc_lo_create(double resolution, uint32_t max_iter) { return new LidarOdometry2D(resolution, max_iter); }
void orc_lo_destroy(void* h) { delete (LidarOdometry2D*)h; }
int orc_lo_update(void* h, const double* pts, int n, const double* origin, const double* quat)
{
    PointCloud pc = make_cloud(pts, n, origin, quat);
    return ((LidarOdometry2D*)h)->update(pc) ? 1 : 0;
}
void orc_lo_get_state(void* h, double* state) { se2_to(((LidarOdometry2D*)h)->odom.state, state); }
void orc_lo_counters(void* h, uint64_t* out)
{
    auto* l = (LidarOdometry2D*)h;
    out[0] = l->last.evals; out[1] = l->last.ray_cells; out[2] = l->last.dm_pops; out[3] = l->last.gn_iters; out[4] = l->removed_patches; out[5] = l->map_updates;
}
void* orc_lo_occ_handle(void* h) { return &((LidarOdometry2D*)h)->occ; }
void* orc_lo_dm_handle(void* h) { return &((LidarOdometry2D*)h)->dm; }
uint64_t orc_slam_removed_patches(void* h) { return ((Slam2D*)h)->removed_patches; }
uint64_t orc_slamp_removed_patches(void* h) { return ((Slam2DProb*)h)->removed_patches; }


void orc_freq_query(void* d, const uint32_t* cells, int n, double* prob, uint8_t* flags) { occ_query(*(FrequencyOccupancyMap*)d, cells, n, prob, flags); }
void orc_prob_query(void* d, const uint32_t* cells, int n, double* prob, uint8_t* flags) { occ_query(*(ProbabilisticOccupancyMap*)d, cells, n, prob, flags); }

}  // extern "C"
extern "C" {
// PFSlam2D::getMemoryUsage() and its (occmem, dmmem) overload, pf_slam2d.cpp:151-176 (the overload sums particle 0's maps P times)
void orc_pf_memory_usage(void* h, uint64_t out[3])
{
    auto* pf = (PFSlam2D*)h;
    out[0] = out[1] = out[2] = 0;
    auto& ps = pf->particles[pf->cur];
    for (size_t i = 0; i < ps.size(); ++i) {
        if (!ps[i].dm || !ps[i].occ) continue;
        out[0] += ps[i].dm->memory(10);
        out[0] += ps[i].occ->memory(4);
        out[1] += ps[0].occ->memory(4);
        out[2] += ps[0].dm->memory(10);
    }
}
// instrumentation: the largest brushfire heap any particle's distance map has held so far
uint64_t orc_pf_peak_queue(void* h)
{
    auto* pf = (PFSlam2D*)h;
    uint64_t m = 0;
    for (auto& p : pf->particles[pf->cur])
        if (p.dm) m = std::max<uint64_t>(m, p.dm->peak_queue);
    return m;
}
}
