// capi.cpp -- the extern "C" boundary declared in include/lama_b200.h.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

// engine.h declares the status codes as an enum; the C header re-states them as macros, so the C++
// headers must come first.
#include "checkpoint.h"
#include "frontend.h"
#include "sdm_io.h"
#include "shard_comm.h"
#include "pgo.h"
#include "tsdm.h"
#include "om3d.h"

#include "../../include/lama_b200.h"

using namespace lama_b200;

namespace lama_b200 { int cuda_device_count(); }

namespace {
thread_local std::string g_err;
int set_err(const std::string& m, int code)
{
    g_err = m;
    return code;
}
// No C++ exception may cross the C boundary (a corrupt file or an allocation failure must come back as a status code, like
// the reference's `return false`): every entry point below is a function-try-block closed by this handler.
#define LAMA_CATCH                                                                                              \
    catch (const std::bad_alloc&) { return set_err("out of host memory", LAMA_ERR_ARG); }                        \
    catch (const std::exception& ex) { return set_err(std::string("exception: ") + ex.what(), LAMA_ERR_ARG); }   \
    catch (...) { return set_err("unknown exception", LAMA_ERR_ARG); }
DeviceOptions dev_from(const lama_device_options& d)
{
    DeviceOptions o;
    o.device     = d.device;
    o.dir_dim    = d.dir_dim > 0 ? d.dir_dim : 64;
    o.pool_slots = d.pool_slots;
    o.max_beams  = d.max_beams > 0 ? d.max_beams : 2048;
    o.timing     = d.timing;
    o.stream     = d.stream;
    return o;
}
void dev_default(lama_device_options* d)
{
    d->device = 0;
    d->dir_dim = 64;
    d->pool_slots = 0;
    d->max_beams = 2048;
    d->timing = 0;
    d->stream = 0;
}
void xyr_of(const SE2& s, double xyr[3])
{
    xyr[0] = s.tx;
    xyr[1] = s.ty;
    xyr[2] = se2_rotation(s);
}
void counters_out(const Counters& c, uint64_t o[6])
{
    o[0] = c.evals; o[1] = c.ray_cells; o[2] = c.dm_pops; o[3] = c.detached; o[4] = c.gn_iters; o[5] = c.resampled;
}
int times_out(Engine* e, double ms[4], uint64_t launches[5])
{
    KernelTimes t = e ? e->times() : KernelTimes();
    if (ms) { ms[0] = t.match_ms; ms[1] = t.raycast_ms; ms[2] = t.brushfire_ms; ms[3] = t.resample_ms; }
    if (launches) {
        launches[0] = t.match_launches; launches[1] = t.raycast_launches; launches[2] = t.brushfire_launches; launches[3] = t.resample_launches;
        launches[4] = t.misc_launches;
    }
    return LAMA_OK;
}
int export_occ(Engine* e, int particle, uint32_t x0, uint32_t y0, int w, int h, uint16_t* occupied, uint16_t* visited, uint8_t* known)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    std::vector<uint32_t> words((size_t)w * h);
    int rc = e->export_window(particle, 0, x0, y0, w, h, words.data(), nullptr);
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    for (size_t i = 0; i < words.size(); ++i) {
        const uint32_t wd = words[i];
        if (occupied) occupied[i] = (uint16_t)occ_occupied(wd);
        if (visited) visited[i] = (uint16_t)occ_visited(wd);
        if (known) known[i] = wd != 0;  // every mutable access counts a visit
    }
    if (known && e->config().known_plane) {   // a pruned cell is {0, 0} and still known: read the known plane
        rc = e->export_bits(particle, 1, x0, y0, w, h, known);
        if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    }
    return LAMA_OK;
}
int export_dm(Engine* e, int particle, bool with_occ, uint32_t x0, uint32_t y0, int w, int h, uint16_t* sqdist, uint8_t* valid, uint8_t* known,
              int16_t* ox, int16_t* oy, uint8_t* queued)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    std::vector<uint32_t> words((size_t)w * h);
    int rc = e->export_window(particle, 1, x0, y0, w, h, words.data(), nullptr);
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    std::vector<uint8_t> occ_known;
    if (with_occ && known && e->config().occupancy_kind == 1) {
        occ_known.resize((size_t)w * h);
        rc = e->export_bits(particle, 1, x0, y0, w, h, occ_known.data());
        if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    } else if (with_occ && known) {
        // The first touch of an occupancy cell always reports "changed" and therefore calls
        // add/removeObstacle, which marks the distance cell known (frequency_occupancy_map.cpp:65-91,
        // dynamic_distance_map.cpp:212-242): distance.known = occupancy.known OR touched by the brushfire.
        std::vector<uint32_t> ow((size_t)w * h);
        rc = e->export_window(particle, 0, x0, y0, w, h, ow.data(), nullptr);
        if (rc != LAMA_OK) return set_err(e->last_error(), rc);
        occ_known.resize(ow.size());
        for (size_t i = 0; i < ow.size(); ++i) occ_known[i] = ow[i] != 0;
    }
    unpack_distance_words(words.data(), occ_known.empty() ? nullptr : occ_known.data(), words.size(), sqdist, valid, known, ox, oy, queued);
    return LAMA_OK;
}
int bounds_out(Engine* e, int particle, int kind, uint32_t mn[2], uint32_t mx[2], int* patches)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    int n = e->bounds(particle, kind, mn, mx);
    if (n < 0) return set_err("bounds failed", LAMA_ERR_ARG);
    if (patches) *patches = n;
    return LAMA_OK;
}
// The reference allocates a distance-map patch wherever an occupancy cell was first touched (see
// export_dm); on the device those cells live only in the occupancy map, so the distance map's
// bounds are the union of both directories.  *patches counts distance patches proper.
int bounds_dm_union(Engine* e, int particle, uint32_t mn[2], uint32_t mx[2], int* patches)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    uint32_t a0[2], a1[2], b0[2], b1[2];
    int nd = e->bounds(particle, 1, a0, a1), no = e->bounds(particle, 0, b0, b1);
    if (nd < 0 || no < 0) return set_err("bounds failed", LAMA_ERR_ARG);
    for (int k = 0; k < 2; ++k) {
        mn[k] = nd && no ? std::min(a0[k], b0[k]) : (nd ? a0[k] : b0[k]);
        mx[k] = nd && no ? std::max(a1[k], b1[k]) : (nd ? a1[k] : b1[k]);
    }
    if (patches) *patches = nd;
    return LAMA_OK;
}

// ---- .sdm files and export images (sdm_io.h) ---------------------------------------------------------------------
struct DmPlanes {
    SdmWindow win;
    std::vector<uint16_t> sqdist;
    std::vector<uint8_t> valid, known, queued;
    std::vector<int16_t> ox, oy;
};
struct OccPlanes {
    SdmWindow win;
    std::vector<uint16_t> occupied, visited;   // frequency maps
    std::vector<float> prob;                   // log-odds maps
    std::vector<uint8_t> known;
};
// kind 1 of a SLAM front end: the reference's distance map also holds the cells first touched through the occupancy map (see export_dm)
int fetch_dm(Engine* e, int particle, bool with_occ, DmPlanes& p)
{
    uint32_t mn[2], mx[2];
    int n = 0;
    int rc = with_occ ? bounds_dm_union(e, particle, mn, mx, &n) : bounds_out(e, particle, 1, mn, mx, &n);
    if (rc != LAMA_OK) return rc;
    if (mx[0] <= mn[0]) { p.win = SdmWindow(); return LAMA_OK; }   // empty map
    p.win.x0 = mn[0]; p.win.y0 = mn[1]; p.win.w = (int)(mx[0] - mn[0]); p.win.h = (int)(mx[1] - mn[1]);
    const size_t cells = (size_t)p.win.w * p.win.h;
    p.sqdist.resize(cells); p.valid.resize(cells); p.known.resize(cells); p.queued.resize(cells); p.ox.resize(cells); p.oy.resize(cells);
    return export_dm(e, particle, with_occ, p.win.x0, p.win.y0, p.win.w, p.win.h, p.sqdist.data(), p.valid.data(), p.known.data(), p.ox.data(), p.oy.data(),
                     p.queued.data());
}
int fetch_occ(Engine* e, int particle, OccPlanes& p)
{
    uint32_t mn[2], mx[2];
    int n = 0;
    int rc = bounds_out(e, particle, 0, mn, mx, &n);
    if (rc != LAMA_OK) return rc;
    if (mx[0] <= mn[0]) { p.win = SdmWindow(); return LAMA_OK; }
    p.win.x0 = mn[0]; p.win.y0 = mn[1]; p.win.w = (int)(mx[0] - mn[0]); p.win.h = (int)(mx[1] - mn[1]);
    const size_t cells = (size_t)p.win.w * p.win.h;
    p.known.resize(cells);
    if (e->config().occupancy_kind == 1) {
        p.prob.resize(cells);
        rc = e->export_window(particle, 0, p.win.x0, p.win.y0, p.win.w, p.win.h, reinterpret_cast<uint32_t*>(p.prob.data()), nullptr);
        if (rc == LAMA_OK) rc = e->export_bits(particle, 1, p.win.x0, p.win.y0, p.win.w, p.win.h, p.known.data());
        return rc == LAMA_OK ? rc : set_err(e->last_error(), rc);
    }
    p.occupied.resize(cells); p.visited.resize(cells);
    return export_occ(e, particle, p.win.x0, p.win.y0, p.win.w, p.win.h, p.occupied.data(), p.visited.data(), p.known.data());
}
// OccupancyMap::{getProbability, isFree, isOccupied, isUnknown}(Vector3ui) of n cells (frequency_occupancy_map.cpp:110-172,
// probabilistic_occupancy_map.cpp:38-41,125-175); flags bit 0 free, bit 1 occupied, bit 2 unknown
int occupancy_query(Engine* e, int particle, const uint32_t* cells, int n, double* prob, uint8_t* flags)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    if (n < 0 || (n && (!cells || !prob || !flags))) return set_err("bad argument", LAMA_ERR_ARG);
    std::vector<uint32_t> words((size_t)n);
    std::vector<uint8_t> fl((size_t)n);
    int rc = e->gather_cells(particle, 0, cells, n, words.data(), fl.data());
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    const bool logodds = e->config().occupancy_kind == 1;
    const double thr = e->logodds_threshold();
    auto prob_of = [](float l) -> float { return 1.0 - 1.0 / (1.0 + std::exp(l)); };   // probabilistic_occupancy_map.cpp:38-41 (float in, float out)
    for (int i = 0; i < n; ++i) {
        if (logodds) {
            const bool known = (fl[i] & 2) != 0;
            float l;
            std::memcpy(&l, &words[i], 4);
            prob[i]  = known ? prob_of(l) : prob_of((float)thr);
            flags[i] = (uint8_t)((known && (double)l < thr ? 1 : 0) | (known && (double)l > thr ? 2 : 0) | (!known || (double)l == thr ? 4 : 0));
        } else {
            const bool known = e->config().known_plane ? (fl[i] & 2) != 0 : words[i] != 0;   // every mutable access counts a visit
            const uint32_t occ = occ_occupied(words[i]), vis = occ_visited(words[i]);
            const double p = vis == 0 ? 0.25 : ((double)occ) / ((double)vis);   // frequency_occupancy_map.cpp:40-45
            prob[i]  = known ? p : 0.25;
            flags[i] = (uint8_t)((known && p < 0.25 ? 1 : 0) | (known && p > 0.25 ? 2 : 0) | (!known || vis == 0 ? 4 : 0));
        }
    }
    return LAMA_OK;
}
// kind 0: occupancy map, kind 1: distance map
int write_map(Engine* e, int particle, int kind, bool slam_frontend, const char* path)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    if (!path || kind < 0 || kind > 1) return set_err("bad argument", LAMA_ERR_ARG);
    SdmFile f;
    const float res = (float)e->config().resolution;   // Map::write stores a float (map.cpp:502)
    if (kind == 1) {
        DmPlanes p;
        int rc = fetch_dm(e, particle, slam_frontend, p);
        if (rc != LAMA_OK) return rc;
        sdm_from_distance(p.win, res, e->max_sqdist(), p.sqdist.data(), p.valid.data(), p.known.data(), p.ox.data(), p.oy.data(), p.queued.data(), f);
    } else {
        OccPlanes p;
        int rc = fetch_occ(e, particle, p);
        if (rc != LAMA_OK) return rc;
        if (e->config().occupancy_kind == 1) sdm_from_logodds(p.win, res, p.prob.data(), p.known.data(), f);
        else sdm_from_frequency(p.win, res, p.occupied.data(), p.visited.data(), p.known.data(), f);
    }
    std::string err;
    if (!sdm_write(path, f, err)) return set_err(err, LAMA_ERR_ARG);
    return LAMA_OK;
}
// grey image of sdm::export_to_png; pixels == NULL: only the dimensions
int export_image(Engine* e, int particle, int kind, bool slam_frontend, uint8_t* pixels, size_t cap, int dims[2])
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    if (!dims || kind < 0 || kind > 1) return set_err("bad argument", LAMA_ERR_ARG);
    if (kind == 1) {
        DmPlanes p;
        int rc = fetch_dm(e, particle, slam_frontend, p);
        if (rc != LAMA_OK) return rc;
        dims[0] = p.win.w; dims[1] = p.win.h;
        if (!pixels) return LAMA_OK;
        if (cap < (size_t)p.win.w * p.win.h) return set_err("image buffer too small", LAMA_ERR_ARG);
        sdm_distance_image(p.win, p.sqdist.data(), p.valid.data(), p.known.data(), e->max_sqdist(), e->config().resolution, pixels);
        return LAMA_OK;
    }
    OccPlanes p;
    int rc = fetch_occ(e, particle, p);
    if (rc != LAMA_OK) return rc;
    dims[0] = p.win.w; dims[1] = p.win.h;
    if (!pixels) return LAMA_OK;
    if (cap < (size_t)p.win.w * p.win.h) return set_err("image buffer too small", LAMA_ERR_ARG);
    if (e->config().occupancy_kind == 1) sdm_occupancy_image_logodds(p.win, p.prob.data(), p.known.data(), e->logodds_threshold(), pixels);
    else sdm_occupancy_image_frequency(p.win, p.occupied.data(), p.visited.data(), p.known.data(), pixels);
    return LAMA_OK;
}
}  // namespace

struct lama_pf { PFSlam2D* p; };
struct lama_slam { Slam2D* s; bool owned = true; };   // borrowed (owned = false): the inner Slam2D of a lama_graph
struct lama_dm { DistanceMapDev* d; bool owned; };
struct lama_om { OccupancyMapDev* m; bool owned; };
struct lama_loc { Loc2D* l; lama_dm dm; };
// om / coarse: the borrowed handles of the generated maps; the graph recreates a map in place, so a handle it returned earlier
// follows the newest map
struct lama_graph { GraphSlam2D* g; lama_slam slam; lama_om om{nullptr, false}; lama_dm coarse{nullptr, false}; };

extern "C" {

const char* lama_last_error(void) { return g_err.c_str(); }
const char* lama_version(void) { return "lama_b200 0.1 sm_90a"; }
int lama_device_count(void) { return lama_b200::cuda_device_count(); }

// ---- PFSlam2D -------------------------------------------------------------------------------------------
int lama_pf_options_default(lama_pf_options* o)
try {
    if (!o) return set_err("null options", LAMA_ERR_ARG);
    std::memset(o, 0, sizeof(*o));
    o->particles = 1;
    o->srr = 0.1; o->str = 0.2; o->stt = 0.1; o->srt = 0.2;
    o->meas_sigma = 0.05; o->meas_sigma_gain = 3;
    o->trans_thresh = 0.5; o->rot_thresh = 0.5;
    o->l2_max = 0.5;
    o->resolution = 0.05;
    o->patch_size = 32; o->max_iter = 100;
    o->strategy = 0; o->threads = -1; o->seed = 0;
    o->shard_rank = 0; o->shard_count = 1;
    dev_default(&o->dev);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_create(const lama_pf_options* o, lama_pf** out)
try {
    if (!o || !out) return set_err("null argument", LAMA_ERR_ARG);
    PFOptions p;
    p.particles = o->particles; p.srr = o->srr; p.str = o->str; p.stt = o->stt; p.srt = o->srt;
    p.meas_sigma = o->meas_sigma; p.meas_sigma_gain = o->meas_sigma_gain; p.trans_thresh = o->trans_thresh; p.rot_thresh = o->rot_thresh;
    p.l2_max = o->l2_max; p.truncated_ray = o->truncated_ray; p.truncated_range = o->truncated_range; p.resolution = o->resolution;
    p.patch_size = o->patch_size; p.max_iter = o->max_iter; p.strategy = o->strategy; p.threads = o->threads; p.seed = o->seed;
    p.shard_rank = o->shard_rank; p.shard_count = o->shard_count ? o->shard_count : 1;
    p.dev = dev_from(o->dev);
    std::string err;
    PFSlam2D* pf = PFSlam2D::create(p, err);
    if (!pf) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_pf{pf};
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_destroy(lama_pf* h)
try {
    if (!h) return LAMA_OK;
    delete h->p;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_set_prior(lama_pf* h, const double xyr[3])
try {
    if (!h || !xyr) return set_err("null argument", LAMA_ERR_ARG);
    h->p->set_prior(xyr[0], xyr[1], xyr[2]);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_update(lama_pf* h, const double* pts, int n, const double* origin, const double* quat, const double* odom, double stamp, int* did_update)
try {
    if (!h || !pts || !odom) return set_err("null argument", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->p->update(pts, n, origin, quat, odom, stamp, &did);
    if (did_update) *did_update = did ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_stage_scans(lama_pf* h, const double* pts, int n_scans, int n)
try {
    if (!h || !pts) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->p->stage_scans(pts, n_scans, n);
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_update_staged(lama_pf* h, int index, const double* origin, const double* quat, const double* odom, double stamp, int* did_update)
try {
    if (!h || !odom) return set_err("null argument", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->p->update_staged(index, origin, quat, odom, stamp, &did);
    if (did_update) *did_update = did ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_get_traffic(lama_pf* h, uint64_t bytes[2], int reset)
try {
    if (!h || !bytes) return set_err("null argument", LAMA_ERR_ARG);
    h->p->settle_counters();
    Engine* e = h->p->engine();
    bytes[0] = e ? e->h2d_bytes() : 0;
    bytes[1] = e ? e->d2h_bytes() : 0;
    if (e && reset) { e->reset_traffic(); e->reset_times(); }
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_pose(lama_pf* h, double xyr[3])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    xyr_of(h->p->pose((int)h->p->best_particle()), xyr);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_best_particle(lama_pf* h, int* idx)
try {
    if (!h || !idx) return set_err("null argument", LAMA_ERR_ARG);
    *idx = (int)h->p->best_particle();
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_neff(lama_pf* h, double* neff)
try {
    if (!h || !neff) return set_err("null argument", LAMA_ERR_ARG);
    *neff = h->p->neff();
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_particles(lama_pf* h, double* states, double* weights)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    for (uint32_t i = 0; i < h->p->particles(); ++i) {
        if (states) { const SE2& s = h->p->pose(i); states[4 * i] = s.c; states[4 * i + 1] = s.s; states[4 * i + 2] = s.tx; states[4 * i + 3] = s.ty; }
        if (weights) h->p->weights(i, &weights[3 * i]);
    }
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_trajectory(lama_pf* h, int particle, double* xyr, int cap, int* count)
try {
    if (!h || particle < 0 || particle >= (int)h->p->particles()) return set_err("bad particle", LAMA_ERR_ARG);
    std::vector<SE2> t = h->p->has_first_scan() ? h->p->trajectory(particle) : std::vector<SE2>();
    for (int i = 0; i < (int)t.size() && i < cap && xyr; ++i) xyr_of(t[i], &xyr[3 * i]);
    if (count) *count = (int)t.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_last_resample(lama_pf* h, int32_t* idx, int* count)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    const std::vector<int32_t>& v = h->p->last_resample();
    if (idx) std::copy(v.begin(), v.end(), idx);
    if (count) *count = (int)v.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_resample_digest(lama_pf* h, uint64_t out[2])
try {
    if (!h || !out) return set_err("null argument", LAMA_ERR_ARG);
    h->p->resample_digest(out);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_summary(lama_pf* h, double ms[4])
try {
    if (!h || !ms) return set_err("null argument", LAMA_ERR_ARG);
    h->p->summary_ms(ms);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_memory_usage(lama_pf* h, uint64_t out[3])
try {
    if (!h || !out) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->p->memory_usage(out);
    return rc == LAMA_OK ? LAMA_OK : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_get_timestamps(lama_pf* h, double* stamps, int cap, int* count)
try {
    if (!h || !count || (cap > 0 && !stamps) || cap < 0) return set_err("null argument / negative capacity", LAMA_ERR_ARG);
    const std::vector<double>& t = h->p->timestamps();
    *count = (int)t.size();
    for (int i = 0; i < cap && i < (int)t.size(); ++i) stamps[i] = t[(size_t)i];
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_get_counters(lama_pf* h, uint64_t last[6], uint64_t total[6])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    if (last) counters_out(h->p->last_counters(), last);
    if (total) counters_out(h->p->total_counters(), total);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_kernel_times(lama_pf* h, double ms[4], uint64_t launches[5])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->p->settle_counters();
    return times_out(h->p->engine(), ms, launches);
}
LAMA_CATCH
static int pf_local(lama_pf* h, int particle)
{
    int k = particle - h->p->local_begin();
    return (k < 0 || k >= h->p->local_count()) ? -1 : k;
}
int lama_pf_map_bounds(lama_pf* h, int particle, int kind, uint32_t mn[2], uint32_t mx[2], int* patches)
try {
    if (!h || pf_local(h, particle) < 0) return set_err("particle not resident on this shard", LAMA_ERR_ARG);
    if (kind == 1) return bounds_dm_union(h->p->engine(), pf_local(h, particle), mn, mx, patches);
    return bounds_out(h->p->engine(), pf_local(h, particle), kind, mn, mx, patches);
}
LAMA_CATCH
int lama_pf_export_occupancy(lama_pf* h, int particle, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited, uint8_t* known)
try {
    if (!h || pf_local(h, particle) < 0) return set_err("particle not resident on this shard", LAMA_ERR_ARG);
    return export_occ(h->p->engine(), pf_local(h, particle), x0, y0, w, hgt, occupied, visited, known);
}
LAMA_CATCH
int lama_pf_distance(lama_pf* h, int particle, const double* pts, int n, double* dist, double* grad)
try {
    if (!h || !pts || !dist) return set_err("null argument", LAMA_ERR_ARG);
    Engine* e = h->p->engine();
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    int rc = e->dm_distance(pf_local(h, particle), pts, n, dist, grad);
    return rc == LAMA_OK ? rc : set_err(e->last_error(), rc);
}
LAMA_CATCH
int lama_pf_occupancy_query(lama_pf* h, int particle, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return occupancy_query(h->p->engine(), pf_local(h, particle), cells_xy, n, prob, flags);
}
LAMA_CATCH
int lama_pf_write_map(lama_pf* h, int particle, int kind, const char* path)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return write_map(h->p->engine(), pf_local(h, particle), kind, true, path);
}
LAMA_CATCH
int lama_pf_export_image(lama_pf* h, int particle, int kind, uint8_t* pixels, size_t cap, int dims[2])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return export_image(h->p->engine(), pf_local(h, particle), kind, true, pixels, cap, dims);
}
LAMA_CATCH
int lama_pf_export_distance(lama_pf* h, int particle, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid, uint8_t* known,
                            int16_t* ox, int16_t* oy, uint8_t* queued)
try {
    if (!h || pf_local(h, particle) < 0) return set_err("particle not resident on this shard", LAMA_ERR_ARG);
    return export_dm(h->p->engine(), pf_local(h, particle), true, x0, y0, w, hgt, sqdist, valid, known, ox, oy, queued);
}
LAMA_CATCH
int lama_pf_shard_begin(lama_pf* h, const double* pts, int n, const double* origin, const double* quat, const double* odom, double stamp,
                        int* did_update, double* local_out)
try {
    if (!h || !pts || !odom || !local_out) return set_err("null argument", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->p->shard_begin(pts, n, origin, quat, odom, stamp, &did, local_out);
    if (did_update) *did_update = did ? (h->p->last_counters().evals ? 2 : 1) : 0;  // 2 = matched, finish/map pending; 1 = first scan
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_shard_finish(lama_pf* h, const double* all_results, int* resampled, int32_t* idx)
try {
    if (!h || !all_results || !resampled || !idx) return set_err("null argument", LAMA_ERR_ARG);
    bool r = false;
    int rc = h->p->shard_finish(all_results, &r, idx);
    *resampled = r ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_shard_apply(lama_pf* h, const int32_t* idx)
try {
    // single-rank form: ancestors are the global indices themselves.  Multi-rank callers use
    // lama_pf_shard_apply_local below after staging remote ancestors with lama_pf_particle_unpack.
    if (!h || !idx) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->p->shard_apply(idx, idx + h->p->local_begin());
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_shard_apply_local(lama_pf* h, const int32_t* idx, const int32_t* local_src)
try {
    if (!h || !idx || !local_src) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->p->shard_apply(idx, local_src);
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_shard_map_update(lama_pf* h)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    int rc = h->p->shard_map_update();
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_shard_unique_id(uint8_t id[128])
try {
    if (!id) return set_err("null argument", LAMA_ERR_ARG);
    std::string err;
    return shard_unique_id(id, err) == 0 ? LAMA_OK : set_err(err, LAMA_ERR_CUDA);
}
LAMA_CATCH
int lama_pf_shard_connect(lama_pf* h, const uint8_t id[128])
try {
    if (!h || !id) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->p->shard_connect(id);
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_shard_stats(lama_pf* h, uint64_t out[2])
try {
    if (!h || !out) return set_err("null argument", LAMA_ERR_ARG);
    h->p->shard_stats(out);
    return LAMA_OK;
}
LAMA_CATCH
int lama_pf_particle_pack_size(lama_pf* h, int slot, size_t* bytes)
try {
    if (!h || !bytes || !h->p->engine()) return set_err("bad argument", LAMA_ERR_ARG);
    int rc = h->p->engine()->pack_size(slot, bytes);
    return rc == LAMA_OK ? rc : set_err(h->p->engine()->last_error(), rc);
}
LAMA_CATCH
int lama_pf_particle_pack(lama_pf* h, int slot, void* buf, size_t cap, size_t* used)
try {
    if (!h || !buf || !used || !h->p->engine()) return set_err("bad argument", LAMA_ERR_ARG);
    int rc = h->p->engine()->pack(slot, buf, cap, used);
    return rc == LAMA_OK ? rc : set_err(h->p->engine()->last_error(), rc);
}
LAMA_CATCH
int lama_pf_particle_unpack(lama_pf* h, int slot, const void* buf, size_t bytes)
try {
    if (!h || !buf || !h->p->engine()) return set_err("bad argument", LAMA_ERR_ARG);
    int rc = h->p->engine()->unpack(slot, buf, bytes);
    return rc == LAMA_OK ? rc : set_err(h->p->engine()->last_error(), rc);
}
LAMA_CATCH

// ---- Slam2D ---------------------------------------------------------------------------------------------
namespace {
SlamOptions slam_from(const lama_slam_options* o)
{
    SlamOptions s;
    s.trans_thresh = o->trans_thresh; s.rot_thresh = o->rot_thresh; s.l2_max = o->l2_max; s.truncated_ray = o->truncated_ray;
    s.transient_map = o->transient_map != 0; s.lidar_odometry = o->lidar_odometry != 0;
    s.truncated_range = o->truncated_range; s.resolution = o->resolution; s.patch_size = o->patch_size; s.max_iter = o->max_iter;
    s.strategy = o->strategy; s.occupancy = o->occupancy; s.dev = dev_from(o->dev);
    return s;
}
}  // namespace
int lama_slam_options_default(lama_slam_options* o)
try {
    if (!o) return set_err("null options", LAMA_ERR_ARG);
    std::memset(o, 0, sizeof(*o));
    o->trans_thresh = 0.5; o->rot_thresh = 0.5; o->l2_max = 0.5; o->resolution = 0.05;
    o->patch_size = 32; o->max_iter = 100; o->strategy = 0;
    dev_default(&o->dev);
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_create(const lama_slam_options* o, lama_slam** out)
try {
    if (!o || !out) return set_err("null argument", LAMA_ERR_ARG);
    const SlamOptions s = slam_from(o);
    std::string err;
    Slam2D* sl = Slam2D::create(s, err);
    if (!sl) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_slam{sl};
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_destroy(lama_slam* h)
try {
    if (!h || !h->owned) return LAMA_OK;
    delete h->s;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_set_pose(lama_slam* h, const double xyr[3])
try {
    if (!h || !xyr) return set_err("null argument", LAMA_ERR_ARG);
    h->s->set_pose(xyr[0], xyr[1], xyr[2]);
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_get_map_stats(lama_slam* h, uint64_t stats[2])
try {
    if (!h || !stats) return set_err("null argument", LAMA_ERR_ARG);
    stats[0] = h->s->map_updates();
    stats[1] = h->s->removed_patches();
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_update(lama_slam* h, const double* pts, int n, const double* origin, const double* quat, const double* odom, double stamp, int* did_update)
try {
    if (!h || !pts) return set_err("null argument", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->s->update(pts, n, origin, quat, odom, stamp, &did);
    if (did_update) *did_update = did ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->s->error(), rc);
}
LAMA_CATCH
int lama_slam_get_pose(lama_slam* h, double xyr[3])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    xyr_of(h->s->pose(), xyr);
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_get_state(lama_slam* h, double st[4])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    const SE2& s = h->s->pose();
    st[0] = s.c; st[1] = s.s; st[2] = s.tx; st[3] = s.ty;
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_get_processed_cells(lama_slam* h, uint32_t* n)
try {
    if (!h || !n) return set_err("null argument", LAMA_ERR_ARG);
    *n = h->s->processed_cells();
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_get_counters(lama_slam* h, uint64_t last[6], uint64_t total[6])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    if (last) counters_out(h->s->last_counters(), last);
    if (total) counters_out(h->s->total_counters(), total);
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_kernel_times(lama_slam* h, double ms[4], uint64_t launches[5])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return times_out(h->s->engine(), ms, launches);
}
LAMA_CATCH
int lama_slam_map_bounds(lama_slam* h, int kind, uint32_t mn[2], uint32_t mx[2], int* patches)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    if (kind == 1) return bounds_dm_union(h->s->engine(), 0, mn, mx, patches);
    return bounds_out(h->s->engine(), 0, kind, mn, mx, patches);
}
LAMA_CATCH
int lama_slam_export_occupancy(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited, uint8_t* known)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return export_occ(h->s->engine(), 0, x0, y0, w, hgt, occupied, visited, known);
}
LAMA_CATCH
int lama_slam_distance(lama_slam* h, const double* pts, int n, double* dist, double* grad)
try {
    if (!h || !pts || !dist) return set_err("null argument", LAMA_ERR_ARG);
    Engine* e = h->s->engine();
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    int rc = e->dm_distance(0, pts, n, dist, grad);
    return rc == LAMA_OK ? rc : set_err(e->last_error(), rc);
}
LAMA_CATCH
int lama_slam_occupancy_query(lama_slam* h, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return occupancy_query(h->s->engine(), 0, cells_xy, n, prob, flags);
}
LAMA_CATCH
int lama_w2m(double resolution, const double* pts_xyz, int n, uint32_t* cells_xy)
try {
    if (!(resolution > 0) || n < 0 || (n && (!pts_xyz || !cells_xy))) return set_err("bad argument", LAMA_ERR_ARG);
    const double scale = 1.0 / resolution;
    for (int i = 0; i < n; ++i) {
        cells_xy[2 * i]     = w2m(pts_xyz[3 * i], scale);
        cells_xy[2 * i + 1] = w2m(pts_xyz[3 * i + 1], scale);
    }
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_write_map(lama_slam* h, int kind, const char* path)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return write_map(h->s->engine(), 0, kind, true, path);
}
LAMA_CATCH
int lama_slam_export_image(lama_slam* h, int kind, uint8_t* pixels, size_t cap, int dims[2])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return export_image(h->s->engine(), 0, kind, true, pixels, cap, dims);
}
LAMA_CATCH
int lama_slam_export_logodds(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, float* logodds, uint8_t* known)
try {
    if (!h || !logodds) return set_err("null argument", LAMA_ERR_ARG);
    Engine* e = h->s->engine();
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    if (e->config().occupancy_kind != 1) return set_err("this Slam2D uses the frequency occupancy map", LAMA_ERR_STATE);
    static_assert(sizeof(float) == 4, "float cells");
    int rc = e->export_window(0, 0, x0, y0, w, hgt, reinterpret_cast<uint32_t*>(logodds), nullptr);
    if (rc == LAMA_OK && known) rc = e->export_bits(0, 1, x0, y0, w, hgt, known);
    return rc == LAMA_OK ? rc : set_err(e->last_error(), rc);
}
LAMA_CATCH
int lama_slam_export_distance(lama_slam* h, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox,
                              int16_t* oy, uint8_t* queued)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return export_dm(h->s->engine(), 0, true, x0, y0, w, hgt, sqdist, valid, known, ox, oy, queued);
}
LAMA_CATCH

// ---- distance map grid interface --------------------------------------------------------------------------
int lama_dm_create(double resolution, uint32_t patch_size, double l2_max, const double center_xy[2], const lama_device_options* dev, lama_dm** out)
try {
    if (!out) return set_err("null argument", LAMA_ERR_ARG);
    lama_device_options d;
    if (dev) d = *dev; else dev_default(&d);
    std::string err;
    DistanceMapDev* m = DistanceMapDev::create(resolution, patch_size, l2_max, center_xy ? center_xy[0] : 0.0, center_xy ? center_xy[1] : 0.0, dev_from(d), err);
    if (!m) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_dm{m, true};
    return LAMA_OK;
}
LAMA_CATCH
int lama_dm_destroy(lama_dm* dm)
try {
    if (!dm) return LAMA_OK;
    if (dm->owned) {
        delete dm->d;
        delete dm;
    }
    return LAMA_OK;
}
LAMA_CATCH
int lama_dm_max_sqdist(lama_dm* dm, uint32_t* v)
try {
    if (!dm || !v) return set_err("null argument", LAMA_ERR_ARG);
    *v = dm->d->engine()->max_sqdist();
    return LAMA_OK;
}
LAMA_CATCH
int lama_dm_add_obstacles(lama_dm* dm, const uint32_t* cells, int n)
try {
    if (!dm || (!cells && n)) return set_err("null argument", LAMA_ERR_ARG);
    return dm->d->add(cells, n, true);
}
LAMA_CATCH
int lama_dm_remove_obstacles(lama_dm* dm, const uint32_t* cells, int n)
try {
    if (!dm || (!cells && n)) return set_err("null argument", LAMA_ERR_ARG);
    return dm->d->add(cells, n, false);
}
LAMA_CATCH
int lama_dm_update(lama_dm* dm, uint32_t* processed)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    int rc = dm->d->update(processed);
    return rc == LAMA_OK ? rc : set_err(dm->d->error(), rc);
}
LAMA_CATCH
int lama_dm_distance(lama_dm* dm, const double* pts, int n, double* dist, double* grad)
try {
    if (!dm || !pts || !dist) return set_err("null argument", LAMA_ERR_ARG);
    int rc = dm->d->flush_if_pending();
    if (rc == LAMA_OK) rc = dm->d->engine()->dm_distance(0, pts, n, dist, grad);
    return rc == LAMA_OK ? rc : set_err(dm->d->engine()->last_error(), rc);
}
LAMA_CATCH
int lama_dm_bounds(lama_dm* dm, uint32_t mn[2], uint32_t mx[2], int* patches)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    return bounds_out(dm->d->engine(), 0, 1, mn, mx, patches);
}
LAMA_CATCH
int lama_dm_export(lama_dm* dm, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* sqdist, uint8_t* valid, uint8_t* known, int16_t* ox, int16_t* oy,
                   uint8_t* queued)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    return export_dm(dm->d->engine(), 0, false, x0, y0, w, hgt, sqdist, valid, known, ox, oy, queued);
}
LAMA_CATCH
int lama_dm_write(lama_dm* dm, const char* path)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    int rc = dm->d->flush_if_pending();
    if (rc != LAMA_OK) return set_err(dm->d->error(), rc);
    return write_map(dm->d->engine(), 0, 1, false, path);
}
LAMA_CATCH
int lama_dm_export_image(lama_dm* dm, uint8_t* pixels, size_t cap, int dims[2])
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    int rc = dm->d->flush_if_pending();
    if (rc != LAMA_OK) return set_err(dm->d->error(), rc);
    return export_image(dm->d->engine(), 0, 1, false, pixels, cap, dims);
}
LAMA_CATCH
// Map::read into an EMPTY device distance map (map.cpp:531-575).  The file must have been written at this map's
// resolution and maximum distance (the reference adopts the file's values; the device map's are fixed at creation).
int lama_dm_read(lama_dm* dm, const char* path)
try {
    if (!dm || !path) return set_err("null argument", LAMA_ERR_ARG);
    Engine* e = dm->d->engine();
    SdmFile f;
    std::string err;
    if (!sdm_read(path, sizeof(SdmDistanceCell), 4, f, err)) return set_err(err, LAMA_ERR_ARG);
    uint32_t max_sqdist = 0;
    std::memcpy(&max_sqdist, f.params.data(), 4);
    if (max_sqdist != e->max_sqdist()) return set_err("the file's max_sqdist differs from this map's l2_max", LAMA_ERR_ARG);
    if (f.header.resolution != (float)e->config().resolution) return set_err("the file's resolution differs from this map's", LAMA_ERR_ARG);
    SdmWindow win;
    if (!sdm_window_of(f, win)) return LAMA_OK;
    {   // the patch ids come from the file: the window they span must lie inside this map's directory window before it is sized
        const DirWindow dw = e->window();
        const int64_t px0 = (int64_t)(win.x0 >> kPatchLog2) - dw.base_px, py0 = (int64_t)(win.y0 >> kPatchLog2) - dw.base_py;
        if (px0 < 0 || py0 < 0 || px0 + (win.w >> kPatchLog2) > dw.dim || py0 + (win.h >> kPatchLog2) > dw.dim)
            return set_err("the file's patches lie outside this map's directory window", LAMA_ERR_WINDOW);
    }
    DmPlanes p;
    const size_t cells = (size_t)win.w * win.h;
    p.sqdist.resize(cells); p.valid.resize(cells); p.known.resize(cells); p.queued.resize(cells); p.ox.resize(cells); p.oy.resize(cells);
    sdm_to_distance(f, win, p.sqdist.data(), p.valid.data(), p.known.data(), p.ox.data(), p.oy.data(), p.queued.data());
    return lama_dm_import(dm, win.x0, win.y0, win.w, win.h, p.sqdist.data(), p.valid.data(), p.known.data(), p.ox.data(), p.oy.data(), p.queued.data());
}
LAMA_CATCH
int lama_dm_import(lama_dm* dm, uint32_t x0, uint32_t y0, int w, int hgt, const uint16_t* sqdist, const uint8_t* valid, const uint8_t* known,
                   const int16_t* ox, const int16_t* oy, const uint8_t* queued)
try {
    if (!dm || !sqdist || !valid || !known) return set_err("null argument", LAMA_ERR_ARG);
    std::vector<uint32_t> words((size_t)w * hgt);
    for (size_t i = 0; i < words.size(); ++i) {
        if (!known[i]) { words[i] = 0; continue; }
        words[i] = dm_pack(sqdist[i], ox ? ox[i] : 0, oy ? oy[i] : 0, valid[i] != 0, queued && queued[i]);
    }
    int rc = dm->d->engine()->import_window(0, 1, x0, y0, w, hgt, words.data());
    return rc == LAMA_OK ? rc : set_err(dm->d->engine()->last_error(), rc);
}
LAMA_CATCH
int lama_dm_match_normal_equations(lama_dm* dm, const double* pts, int n, const double* origin, const double* quat, const double* states, int count,
                                   int robust_kind, double robust_param, double meas_sigma, double* out)
try {
    if (!dm || !pts || !states || !out || count < 1) return set_err("bad argument", LAMA_ERR_ARG);
    Engine* e = dm->d->engine();
    int rc = dm->d->flush_if_pending();
    if (rc == LAMA_OK) rc = e->set_scan(pts, n, origin, quat, 0, 0);
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    SolverOptions so = make_solver(0, 0);
    so.robust_kind = robust_kind;
    so.robust_param = robust_param;
    std::vector<SE2> st((size_t)count);
    for (int i = 0; i < count; ++i) st[i] = SE2{states[4 * i], states[4 * i + 1], states[4 * i + 2], states[4 * i + 3]};
    std::vector<HostMatchResult> res((size_t)count);
    rc = e->match(st.data(), count, 0, true, so, meas_sigma, 1, res.data());
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    for (int i = 0; i < count; ++i) std::memcpy(out + (size_t)i * kNumSums, res[i].sums, sizeof(double) * kNumSums);
    return LAMA_OK;
}
LAMA_CATCH
int lama_dm_match_solve(lama_dm* dm, const double* pts, int n, const double* origin, const double* quat, double* states, int count, int strategy,
                        int robust_kind, double robust_param, uint32_t max_iter, uint32_t* stats, double* sums)
try {
    if (!dm || !pts || !states || count < 1) return set_err("bad argument", LAMA_ERR_ARG);
    Engine* e = dm->d->engine();
    int rc = dm->d->flush_if_pending();
    if (rc == LAMA_OK) rc = e->set_scan(pts, n, origin, quat, 0, 0);
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    SolverOptions so = make_solver(strategy, max_iter);
    so.robust_kind = robust_kind;
    so.robust_param = robust_param;
    std::vector<SE2> st((size_t)count);
    for (int i = 0; i < count; ++i) st[i] = SE2{states[4 * i], states[4 * i + 1], states[4 * i + 2], states[4 * i + 3]};
    std::vector<HostMatchResult> res((size_t)count);
    rc = e->match(st.data(), count, 0, true, so, 0.05, 0, res.data());
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    for (int i = 0; i < count; ++i) {
        states[4 * i] = res[i].state.c; states[4 * i + 1] = res[i].state.s; states[4 * i + 2] = res[i].state.tx; states[4 * i + 3] = res[i].state.ty;
        if (stats) { stats[2 * i] = res[i].iterations; stats[2 * i + 1] = res[i].evals_ref; }
        if (sums) std::memcpy(sums + (size_t)i * kNumSums, res[i].sums, sizeof(double) * kNumSums);
    }
    return LAMA_OK;
}
LAMA_CATCH

// ---- SimplePGO (src/simple_pgo.cpp:48-105) -----------------------------------------------------------------------------------------------------
int lama_pgo_optimize(int device, double* nodes_xyr, int n_nodes, const int* edges_from_to, const double* edges_xyr, int n_edges, const int* fixed_nodes,
                      const double* fixed_xyr, int n_fixed, int* status, double report[6])
try {
    if (!nodes_xyr || n_nodes < 1 || n_edges < 0 || n_fixed < 0 || (n_edges && (!edges_from_to || !edges_xyr)) || (n_fixed && (!fixed_nodes || !fixed_xyr)))
        return set_err("bad argument", LAMA_ERR_ARG);
    std::vector<SE2> nodes((size_t)n_nodes);
    for (int i = 0; i < n_nodes; ++i) nodes[(size_t)i] = se2_from_xyr(nodes_xyr[3 * i], nodes_xyr[3 * i + 1], nodes_xyr[3 * i + 2]);
    std::vector<PgoEdge> edges((size_t)n_edges);
    for (int e = 0; e < n_edges; ++e)
        edges[(size_t)e] = PgoEdge{edges_from_to[2 * e], edges_from_to[2 * e + 1], se2_from_xyr(edges_xyr[3 * e], edges_xyr[3 * e + 1], edges_xyr[3 * e + 2])};
    std::vector<PgoFixed> fixed((size_t)n_fixed);
    for (int f = 0; f < n_fixed; ++f) fixed[(size_t)f] = PgoFixed{fixed_nodes[f], se2_from_xyr(fixed_xyr[3 * f], fixed_xyr[3 * f + 1], fixed_xyr[3 * f + 2])};
    PgoReport rep;
    std::string err;
    const int rc = pgo_optimize(device, nodes, edges, fixed, rep, err);
    if (rc != LAMA_OK) return set_err(err, rc);
    if (status) *status = rep.status;
    if (report) {
        report[0] = rep.iterations; report[1] = rep.lambda_tries; report[2] = (double)rep.cg_iterations;
        report[3] = rep.initial_error; report[4] = rep.final_error; report[5] = rep.device_ms;
    }
    if (rep.status == 0)
        for (int i = 0; i < n_nodes; ++i) xyr_of(nodes[(size_t)i], nodes_xyr + 3 * i);
    return LAMA_OK;
}
LAMA_CATCH

// ---- LevenbergMarquardtOptimizer over an explicit factor graph (GraphSlam2D's graph goes through the same pgo_optimize_graph) -------------------
int lama_pgo_optimize_graph(int device, double* nodes_xyr, int n_nodes, const int* prior_nodes, const double* prior_xyr, const double* prior_loss, int n_priors,
                            const int* between_from_to, const double* between_xyr, const double* between_loss, int n_betweens, int* status, double report[6],
                            uint8_t* accepted, int accepted_cap, int* n_tries)
try {
    if (!nodes_xyr || n_nodes < 1 || n_priors < 0 || n_betweens < 0 || (n_priors && (!prior_nodes || !prior_xyr || !prior_loss)) ||
        (n_betweens && (!between_from_to || !between_xyr || !between_loss)) || (accepted && accepted_cap < 0))
        return set_err("bad argument", LAMA_ERR_ARG);
    auto loss_of = [](const double* l) { return PgoLoss{{l[0], l[1], l[2]}, l[3]}; };
    std::vector<SE2> nodes((size_t)n_nodes);
    for (int i = 0; i < n_nodes; ++i) nodes[(size_t)i] = se2_from_xyr(nodes_xyr[3 * i], nodes_xyr[3 * i + 1], nodes_xyr[3 * i + 2]);
    std::vector<PgoPrior> priors((size_t)n_priors);
    for (int f = 0; f < n_priors; ++f)
        priors[(size_t)f] = PgoPrior{prior_nodes[f], se2_from_xyr(prior_xyr[3 * f], prior_xyr[3 * f + 1], prior_xyr[3 * f + 2]), loss_of(prior_loss + 4 * f)};
    std::vector<PgoBetween> betweens((size_t)n_betweens);
    for (int f = 0; f < n_betweens; ++f)
        betweens[(size_t)f] = PgoBetween{between_from_to[2 * f], between_from_to[2 * f + 1],
                                         se2_from_xyr(between_xyr[3 * f], between_xyr[3 * f + 1], between_xyr[3 * f + 2]), loss_of(between_loss + 4 * f)};
    PgoReport rep;
    std::string err;
    const int rc = pgo_optimize_graph(device, nodes, priors, betweens, rep, err);
    if (rc != LAMA_OK) return set_err(err, rc);
    if (status) *status = rep.status;
    if (report) {
        report[0] = rep.iterations; report[1] = rep.lambda_tries; report[2] = (double)rep.cg_iterations;
        report[3] = rep.initial_error; report[4] = rep.final_error; report[5] = rep.device_ms;
    }
    if (accepted) std::copy_n(rep.accepted.begin(), std::min<size_t>(rep.accepted.size(), (size_t)accepted_cap), accepted);
    if (n_tries) *n_tries = (int)rep.accepted.size();
    if (rep.status == 0)
        for (int i = 0; i < n_nodes; ++i) xyr_of(nodes[(size_t)i], nodes_xyr + 3 * i);
    return LAMA_OK;
}
LAMA_CATCH

// ---- GraphSlam2D loop-closure front end (src/graph_slam2d.cpp:283-392) ---------------------------------------------------------------------
namespace {
int correlate_on(Engine* e, const DeviceOptions* coarse_dev, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat, const double* pts, int n,
                 const double* origin, const double* quat, const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3], double* rmse)
{
    if (!e) return set_err("no map yet (update() has not been called)", LAMA_ERR_STATE);
    if (!pts || n < 1 || !ref_xyr || !cand_xyr || !between_xyr || !rmse) return set_err("bad argument", LAMA_ERR_ARG);
    const SE2 ref = se2_from_xyr(ref_xyr[0], ref_xyr[1], ref_xyr[2]), cand = se2_from_xyr(cand_xyr[0], cand_xyr[1], cand_xyr[2]);
    SE2 between{1, 0, 0, 0};
    int rc;
    if (coarse_dev) {
        if (!ref_pts || ref_n < 1) return set_err("bad argument", LAMA_ERR_ARG);
        std::string err;
        rc = coarse_correlate_candidate_scan(e, 0, *coarse_dev, ref_pts, ref_n, ref_origin, ref_quat, pts, n, origin, quat, ref, cand, &between, rmse, err);
        if (rc != LAMA_OK) return set_err(err, rc);
    } else {
        rc = correlate_candidate_scan(e, 0, pts, n, origin, quat, ref, cand, &between, rmse);
        if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    }
    xyr_of(between, between_xyr);
    return LAMA_OK;
}
}  // namespace
int lama_loop_closure_candidates(const double* key_xy, int n_keys, int ignore_n_chain_poses, const double query_xy[2], double radius, int max_candidates, int* ids,
                                 int* count)
try {
    if (!key_xy || !query_xy || !ids || !count || n_keys < 0 || max_candidates < 0) return set_err("bad argument", LAMA_ERR_ARG);
    const std::vector<int> v = find_loop_closure_candidates(key_xy, n_keys, ignore_n_chain_poses, query_xy, radius, max_candidates);
    std::copy(v.begin(), v.end(), ids);
    *count = (int)v.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_correlate_candidate_scan(lama_slam* h, const double* pts, int n, const double* origin, const double* quat, const double ref_xyr[3],
                                       const double cand_xyr[3], double between_xyr[3], double* rmse)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    return correlate_on(h->s->engine(), nullptr, nullptr, 0, nullptr, nullptr, pts, n, origin, quat, ref_xyr, cand_xyr, between_xyr, rmse);
}
LAMA_CATCH
int lama_slam_coarse_correlate_candidate_scan(lama_slam* h, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat, const double* pts, int n,
                                              const double* origin, const double* quat, const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3],
                                              double* rmse)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    const DeviceOptions dev = h->s->device_options();
    return correlate_on(h->s->engine(), &dev, ref_pts, ref_n, ref_origin, ref_quat, pts, n, origin, quat, ref_xyr, cand_xyr, between_xyr, rmse);
}
LAMA_CATCH
int lama_dm_correlate_candidate_scan(lama_dm* dm, const double* pts, int n, const double* origin, const double* quat, const double ref_xyr[3],
                                     const double cand_xyr[3], double between_xyr[3], double* rmse)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    int rc = dm->d->flush_if_pending();
    if (rc != LAMA_OK) return set_err(dm->d->error(), rc);
    return correlate_on(dm->d->engine(), nullptr, nullptr, 0, nullptr, nullptr, pts, n, origin, quat, ref_xyr, cand_xyr, between_xyr, rmse);
}
LAMA_CATCH
int lama_dm_coarse_correlate_candidate_scan(lama_dm* dm, const double* ref_pts, int ref_n, const double* ref_origin, const double* ref_quat, const double* pts, int n,
                                            const double* origin, const double* quat, const double ref_xyr[3], const double cand_xyr[3], double between_xyr[3],
                                            double* rmse)
try {
    if (!dm) return set_err("null handle", LAMA_ERR_ARG);
    int rc = dm->d->flush_if_pending();
    if (rc != LAMA_OK) return set_err(dm->d->error(), rc);
    DeviceOptions dev;
    dev.device = dm->d->engine()->config().device;
    return correlate_on(dm->d->engine(), &dev, ref_pts, ref_n, ref_origin, ref_quat, pts, n, origin, quat, ref_xyr, cand_xyr, between_xyr, rmse);
}
LAMA_CATCH
int lama_dm_match_error(lama_dm* dm, const double* pts, int n, const double* origin, const double* quat, const double* states, int count, double* rmse)
try {
    if (!dm || !pts || !states || !rmse || count < 1) return set_err("bad argument", LAMA_ERR_ARG);
    Engine* e = dm->d->engine();
    int rc = dm->d->flush_if_pending();
    if (rc == LAMA_OK) rc = e->set_scan(pts, n, origin, quat, 0, 0);
    if (rc != LAMA_OK) return set_err(e->last_error(), rc);
    std::vector<SE2> st((size_t)count);
    for (int i = 0; i < count; ++i) st[i] = SE2{states[4 * i], states[4 * i + 1], states[4 * i + 2], states[4 * i + 3]};
    rc = e->match_error(st.data(), count, 0, true, rmse);
    return rc == LAMA_OK ? rc : set_err(e->last_error(), rc);
}
LAMA_CATCH

// ---- Loc2D ------------------------------------------------------------------------------------------------
int lama_loc_options_default(lama_loc_options* o)
try {
    if (!o) return set_err("null options", LAMA_ERR_ARG);
    std::memset(o, 0, sizeof(*o));
    o->trans_thresh = 0.5; o->rot_thresh = 0.5; o->l2_max = 1.0; o->resolution = 0.05;
    o->patch_size = 32; o->max_iter = 100; o->strategy = 0;
    o->gloc_particles = 3000; o->gloc_iters = 10; o->gloc_thresh = 0.15; o->cov_blend = 0.0;  // loc2d.cpp:53-57
    dev_default(&o->dev);
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_create(const lama_loc_options* o, lama_loc** out)
try {
    if (!o || !out) return set_err("null argument", LAMA_ERR_ARG);
    LocOptions l;
    l.trans_thresh = o->trans_thresh; l.rot_thresh = o->rot_thresh; l.l2_max = o->l2_max; l.resolution = o->resolution;
    l.patch_size = o->patch_size; l.max_iter = o->max_iter; l.strategy = o->strategy; l.center_x = o->center_xy[0]; l.center_y = o->center_xy[1];
    l.gloc_particles = o->gloc_particles; l.gloc_iters = o->gloc_iters; l.gloc_thresh = o->gloc_thresh; l.cov_blend = o->cov_blend;
    l.dev = dev_from(o->dev);
    std::string err;
    Loc2D* loc = Loc2D::create(l, err);
    if (!loc) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_loc{loc, lama_dm{loc->distance_map(), false}};
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_destroy(lama_loc* h)
try {
    if (!h) return LAMA_OK;
    delete h->l;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_distance_map(lama_loc* h, lama_dm** dm)
try {
    if (!h || !dm) return set_err("null argument", LAMA_ERR_ARG);
    *dm = &h->dm;
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_set_pose(lama_loc* h, const double xyr[3])
try {
    if (!h || !xyr) return set_err("null argument", LAMA_ERR_ARG);
    h->l->set_pose(xyr[0], xyr[1], xyr[2]);
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_update(lama_loc* h, const double* pts, int n, const double* origin, const double* quat, const double* odom, double stamp, int force,
                    int* did_update)
try {
    if (!h || !pts || !odom) return set_err("null argument", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->l->update(pts, n, origin, quat, odom, stamp, force != 0, &did);
    if (did_update) *did_update = did ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->l->error(), rc);
}
LAMA_CATCH
int lama_loc_get_pose(lama_loc* h, double xyr[3])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    xyr_of(h->l->pose(), xyr);
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_get_state(lama_loc* h, double st[4])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    const SE2& s = h->l->pose();
    st[0] = s.c; st[1] = s.s; st[2] = s.tx; st[3] = s.ty;
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_get_covar(lama_loc* h, double cov[9])
try {
    if (!h || !cov) return set_err("null argument", LAMA_ERR_ARG);
    std::memcpy(cov, h->l->cov(), sizeof(double) * 9);
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_get_rmse(lama_loc* h, double* rmse)
try {
    if (!h || !rmse) return set_err("null argument", LAMA_ERR_ARG);
    *rmse = h->l->rmse();
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_occupancy_set(lama_loc* h, const uint32_t* cells, int n, int state)
try {
    if (!h || (!cells && n)) return set_err("null argument", LAMA_ERR_ARG);
    for (int i = 0; i < n; ++i) h->l->occupancy_map()->set(cells[2 * i], cells[2 * i + 1], state);
    return LAMA_OK;
}
LAMA_CATCH
// SimpleOccupancyMap::read (Map::read, map.cpp:531-575; int8 cells: -1 free, 0 unknown, 1 occupied)
int lama_loc_occupancy_read(lama_loc* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    SdmFile f;
    std::string err;
    if (!sdm_read(path, 1, 0, f, err)) return set_err(err, LAMA_ERR_ARG);
    // Map::read adopts the file's resolution (map.cpp:549-558); this map's scale is fixed at Init, so a different one is refused
    if (f.header.resolution != (float)h->l->occupancy_map()->resolution()) return set_err("the file's resolution differs from this map's", LAMA_ERR_ARG);
    for (size_t i = 0; i < f.ids.size(); ++i) {
        const uint32_t ax = (uint32_t)(f.ids[i] / 2642244ull) << kPatchLog2, ay = (uint32_t)(f.ids[i] % 2642244ull) << kPatchLog2;
        const int8_t* c = reinterpret_cast<const int8_t*>(f.cells.data() + i * (size_t)kPatchCells);
        const uint64_t* mask = f.masks.data() + i * (kPatchCells / 64);
        for (uint32_t ci = 0; ci < (uint32_t)kPatchCells; ++ci)
            if ((mask[ci >> 6] >> (ci & 63)) & 1ull) h->l->occupancy_map()->set(ax + (ci & (kPatchLen - 1)), ay + (ci >> kPatchLog2), c[ci]);
    }
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_set_seed(lama_loc* h, uint32_t seed)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->l->set_seed(seed);
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_trigger_global_localization(lama_loc* h)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->l->trigger_global_localization();
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_global_localization_active(lama_loc* h, int* active)
try {
    if (!h || !active) return set_err("null argument", LAMA_ERR_ARG);
    *active = h->l->global_localization_active() ? 1 : 0;
    return LAMA_OK;
}
LAMA_CATCH
int lama_loc_get_solve_stats(lama_loc* h, uint32_t stats[2])
try {
    if (!h || !stats) return set_err("null argument", LAMA_ERR_ARG);
    stats[0] = h->l->iterations();
    stats[1] = h->l->evals();
    return LAMA_OK;
}
LAMA_CATCH

// ---- GraphSlam2D (src/graph_slam2d.cpp:104-430) ------------------------------------------------------------------------------------------------
int lama_graph_options_default(lama_graph_options* o)
try {
    if (!o) return set_err("null options", LAMA_ERR_ARG);
    std::memset(o, 0, sizeof(*o));
    int rc = lama_slam_options_default(&o->slam);   // Options : Slam2D::Options (graph_slam2d.h:59-60)
    if (rc != LAMA_OK) return rc;
    o->key_pose_distance = 1.0; o->key_pose_angular_distance = 0.5 * M_PI; o->key_pose_head_delay = 5;   // graph_slam2d.h:62-86
    o->loop_search_max_distance = 10.0; o->loop_search_min_distance = 2.0; o->loop_max_candidates = 5;
    o->loop_closure_scan_rmse = 0.05; o->loop_closure_max_candidates = 10; o->ignore_n_chain_poses = 20;
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_create(const lama_graph_options* o, lama_graph** out)
try {
    if (!o || !out) return set_err("null argument", LAMA_ERR_ARG);
    GraphOptions g;
    g.slam = slam_from(&o->slam);
    g.key_pose_distance = o->key_pose_distance; g.key_pose_angular_distance = o->key_pose_angular_distance; g.key_pose_head_delay = o->key_pose_head_delay;
    g.loop_search_max_distance = o->loop_search_max_distance; g.loop_search_min_distance = o->loop_search_min_distance;
    g.loop_max_candidates = o->loop_max_candidates; g.loop_closure_scan_rmse = o->loop_closure_scan_rmse;
    g.loop_closure_max_candidates = o->loop_closure_max_candidates; g.ignore_n_chain_poses = o->ignore_n_chain_poses;
    if (g.key_pose_head_delay < 0 || g.ignore_n_chain_poses < 0 || g.loop_max_candidates < 0) return set_err("GraphSlam2D: negative count in the options", LAMA_ERR_ARG);
    std::string err;
    GraphSlam2D* gs = GraphSlam2D::create(g, err);
    if (!gs) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_graph{gs, lama_slam{gs->slam(), false}, lama_om{nullptr, false}, lama_dm{nullptr, false}};
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_destroy(lama_graph* h)
try {
    if (!h) return LAMA_OK;
    delete h->g;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_set_pose(lama_graph* h, const double xyr[3])
try {
    if (!h || !xyr) return set_err("null argument", LAMA_ERR_ARG);
    h->g->init(xyr[0], xyr[1], xyr[2]);
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_update(lama_graph* h, const double* pts, int n, const double* origin, const double* quat, const double* odom, double stamp, int* did_update)
try {
    if (!h || !pts || !odom || n < 1) return set_err("null argument or empty scan", LAMA_ERR_ARG);
    bool did = false;
    int rc = h->g->update(pts, n, origin, quat, odom, stamp, &did);
    if (did_update) *did_update = did ? 1 : 0;
    return rc == LAMA_OK ? rc : set_err(h->g->error(), rc);
}
LAMA_CATCH
int lama_graph_get_pose(lama_graph* h, double xyr[3])
try {
    if (!h || !xyr) return set_err("null argument", LAMA_ERR_ARG);
    xyr_of(h->g->pose(), xyr);
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_get_key_poses(lama_graph* h, double* corrected_xyr, double* original_xyr, double* stamps, int cap, int* count)
try {
    if (!h || !count || cap < 0) return set_err("null argument", LAMA_ERR_ARG);
    const auto& k = h->g->key_poses();
    const int m = std::min(cap, (int)k.size());
    for (int i = 0; i < m; ++i) {
        if (corrected_xyr) xyr_of(k[(size_t)i].pose, corrected_xyr + 3 * i);
        if (original_xyr) xyr_of(k[(size_t)i].original, original_xyr + 3 * i);
        if (stamps) stamps[i] = k[(size_t)i].stamp;
    }
    *count = (int)k.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_get_key_cloud(lama_graph* h, int key, double* pts, int cap, double* origin, double* quat, int* count)
try {
    if (!h || !count || cap < 0) return set_err("null argument", LAMA_ERR_ARG);
    const auto& k = h->g->key_poses();
    if (key < 0 || key >= (int)k.size()) return set_err("no such key pose", LAMA_ERR_ARG);
    const auto& kp = k[(size_t)key];
    const int n = (int)(kp.pts.size() / 3);
    if (pts) std::copy_n(kp.pts.begin(), 3 * (size_t)std::min(cap, n), pts);
    if (origin) std::copy_n(kp.origin, 3, origin);
    if (quat) std::copy_n(kp.quat, 4, quat);
    *count = n;
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_get_links(lama_graph* h, int32_t* from_to, int cap, int* count)
try {
    if (!h || !count || cap < 0 || (cap > 0 && !from_to)) return set_err("null argument", LAMA_ERR_ARG);
    const auto& l = h->g->links();
    const int m = std::min(cap, (int)l.size());
    for (int i = 0; i < m; ++i) { from_to[2 * i] = l[(size_t)i].first; from_to[2 * i + 1] = l[(size_t)i].second; }
    *count = (int)l.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_get_last_candidates(lama_graph* h, int32_t* ids, int cap, int* count)
try {
    if (!h || !count || cap < 0 || (cap > 0 && !ids)) return set_err("null argument", LAMA_ERR_ARG);
    const auto& c = h->g->last_candidates();
    std::copy_n(c.begin(), std::min<size_t>(c.size(), (size_t)cap), ids);
    *count = (int)c.size();
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_get_stats(lama_graph* h, uint64_t counts[4], int* last_status, double last_report[6])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    const GraphSlam2D::Stats& s = h->g->stats();
    if (counts) { counts[0] = h->g->key_poses().size(); counts[1] = s.loop_factors; counts[2] = s.optimizations; counts[3] = s.optimizations_ok; }
    if (last_status) *last_status = s.last.status;
    if (last_report) {
        last_report[0] = s.last.iterations; last_report[1] = s.last.lambda_tries; last_report[2] = (double)s.last.cg_iterations;
        last_report[3] = s.last.initial_error; last_report[4] = s.last.final_error; last_report[5] = s.last.device_ms;
    }
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_slam(lama_graph* h, lama_slam** slam)
try {
    if (!h || !slam) return set_err("null argument", LAMA_ERR_ARG);
    *slam = &h->slam;
    return LAMA_OK;
}
LAMA_CATCH
// GraphSlam2D::generateOccupancyMap (graph_slam2d.cpp:131-164)
int lama_graph_generate_occupancy_map(lama_graph* h, int full, lama_om** om)
try {
    if (!h || !om) return set_err("null argument", LAMA_ERR_ARG);
    OccupancyMapDev* m = nullptr;
    int rc = h->g->generate_occupancy_map(full != 0, &m);
    h->om.m = h->g->occupancy_map();   // null until the first successful call
    if (rc != LAMA_OK) return set_err(h->g->error(), rc);
    *om = &h->om;
    return LAMA_OK;
}
LAMA_CATCH
// GraphSlam2D::generateCoarseDistanceMap (graph_slam2d.cpp:166-186)
int lama_graph_generate_coarse_distance_map(lama_graph* h, lama_dm** dm, uint32_t* processed)
try {
    if (!h || !dm) return set_err("null argument", LAMA_ERR_ARG);
    DistanceMapDev* d = nullptr;
    int rc = h->g->generate_coarse_distance_map(&d, processed);
    h->coarse.d = h->g->coarse_distance_map();
    if (rc != LAMA_OK) return set_err(h->g->error(), rc);
    *dm = &h->coarse;
    return LAMA_OK;
}
LAMA_CATCH

// ---- FrequencyOccupancyMap (include/lama/sdm/frequency_occupancy_map.h) -------------------------------------------------------------
namespace {
Engine* om_engine(lama_om* om) { return om && om->m ? om->m->engine() : nullptr; }
}
// FrequencyOccupancyMap(resolution, patch_size) (frequency_occupancy_map.cpp:47-49) on the device, window centred on center_xy
int lama_om_create(double resolution, uint32_t patch_size, const double center_xy[2], const lama_device_options* dev, lama_om** out)
try {
    if (!out) return set_err("null argument", LAMA_ERR_ARG);
    if (!(resolution > 0)) return set_err("resolution must be positive", LAMA_ERR_ARG);
    lama_device_options d;
    if (dev) d = *dev; else dev_default(&d);
    std::string err;
    OccupancyMapDev* m = OccupancyMapDev::create(resolution, patch_size, center_xy ? center_xy[0] : 0.0, center_xy ? center_xy[1] : 0.0, dev_from(d), err);
    if (!m) return set_err(err, lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : LAMA_ERR_ARG);
    *out = new lama_om{m, true};
    return LAMA_OK;
}
LAMA_CATCH
int lama_om_destroy(lama_om* om)
try {
    if (!om || !om->owned) return LAMA_OK;   // a borrowed handle belongs to its lama_graph
    delete om->m;
    delete om;
    return LAMA_OK;
}
LAMA_CATCH
// the loop of graph_slam2d.cpp:135-160 for any posed scans: setOccupied(tf * p) and, with full, setFree along computeRay(so, hit)
int lama_om_insert_scans(lama_om* om, const double* pts_xyz, const int64_t* offsets, int n_scans, const double* origins, const double* quats_xyzw,
                         const double* states, int full, uint64_t* cells)
try {
    if (!om || (n_scans > 0 && (!offsets || !states))) return set_err("null argument", LAMA_ERR_ARG);
    if (!om->m) return set_err("no map yet (generateOccupancyMap has not been called)", LAMA_ERR_STATE);
    if (n_scans < 0) return set_err("negative number of scans", LAMA_ERR_ARG);
    std::vector<SE2> st((size_t)n_scans);
    for (int k = 0; k < n_scans; ++k) st[k] = SE2{states[4 * k], states[4 * k + 1], states[4 * k + 2], states[4 * k + 3]};
    int rc = om->m->insert_scans(pts_xyz, offsets, n_scans, origins, quats_xyzw, st.data(), full != 0, cells);
    return rc == LAMA_OK ? rc : set_err(om->m->error(), rc);
}
LAMA_CATCH
// FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158)
int lama_om_prune(lama_om* om)
try {
    if (!om) return set_err("null handle", LAMA_ERR_ARG);
    if (!om->m) return set_err("no map yet (generateOccupancyMap has not been called)", LAMA_ERR_STATE);
    int rc = om->m->prune();
    return rc == LAMA_OK ? rc : set_err(om->m->error(), rc);
}
LAMA_CATCH
int lama_om_resolution(lama_om* om, double* resolution)
try {
    if (!om || !resolution) return set_err("null argument", LAMA_ERR_ARG);
    Engine* e = om_engine(om);
    if (!e) return set_err("no map yet (generateOccupancyMap has not been called)", LAMA_ERR_STATE);
    *resolution = e->config().resolution;
    return LAMA_OK;
}
LAMA_CATCH
// Map::bounds (map.cpp:139-157) in cells, patch granular
int lama_om_bounds(lama_om* om, uint32_t mn[2], uint32_t mx[2], int* patches)
try {
    if (!om || !mn || !mx) return set_err("null argument", LAMA_ERR_ARG);
    return bounds_out(om_engine(om), 0, 0, mn, mx, patches);
}
LAMA_CATCH
// getProbability / isFree / isOccupied / isUnknown (frequency_occupancy_map.cpp:110-172), flags as lama_pf_occupancy_query
int lama_om_query(lama_om* om, const uint32_t* cells_xy, int n, double* prob, uint8_t* flags)
try {
    if (!om) return set_err("null handle", LAMA_ERR_ARG);
    return occupancy_query(om_engine(om), 0, cells_xy, n, prob, flags);
}
LAMA_CATCH
int lama_om_export(lama_om* om, uint32_t x0, uint32_t y0, int w, int hgt, uint16_t* occupied, uint16_t* visited, uint8_t* known)
try {
    if (!om) return set_err("null handle", LAMA_ERR_ARG);
    if (w < 1 || hgt < 1) return set_err("empty window", LAMA_ERR_ARG);
    return export_occ(om_engine(om), 0, x0, y0, w, hgt, occupied, visited, known);
}
LAMA_CATCH
// Map::write (map.cpp:490-529)
int lama_om_write(lama_om* om, const char* path)
try {
    if (!om || !path) return set_err("null argument", LAMA_ERR_ARG);
    return write_map(om_engine(om), 0, 0, false, path);
}
LAMA_CATCH
// the grey image of sdm::export_to_png (export.cpp:46-96); pixels == NULL: only the dimensions
int lama_om_export_image(lama_om* om, uint8_t* pixels, size_t cap, int dims[2])
try {
    if (!om || !dims) return set_err("null argument", LAMA_ERR_ARG);
    return export_image(om_engine(om), 0, 0, false, pixels, cap, dims);
}
LAMA_CATCH
int lama_om_kernel_times(lama_om* om, double ms[4], uint64_t launches[5])
try {
    if (!om) return set_err("null handle", LAMA_ERR_ARG);
    return times_out(om_engine(om), ms, launches);
}
LAMA_CATCH

// ---- TruncatedSignedDistanceMap (include/lama/sdm/truncated_signed_distance_map.h) -------------------------------------------------
struct lama_tsdm { TsdmDev* t; };
// TruncatedSignedDistanceMap(resolution, patch_size, is3d) (truncated_signed_distance_map.cpp:41-49) on the device
int lama_tsdm_create(double resolution, uint32_t patch_size, int is3d, const double center_xyz[3], const int32_t window_patches[3],
                     const lama_device_options* dev, lama_tsdm** out)
try {
    if (!out) return set_err("null argument", LAMA_ERR_ARG);
    lama_device_options d;
    if (dev) d = *dev; else dev_default(&d);
    std::string err;
    TsdmDev* t = TsdmDev::create(resolution, patch_size, is3d != 0, center_xyz, window_patches, dev_from(d), err);
    if (!t) {
        const bool bad_arg = !(resolution > 0) || patch_size != 32 || err.find("window") != std::string::npos;
        return set_err(err, !bad_arg && lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : (bad_arg ? LAMA_ERR_ARG : LAMA_ERR_CUDA));
    }
    *out = new lama_tsdm{t};
    return LAMA_OK;
}
LAMA_CATCH
int lama_tsdm_destroy(lama_tsdm* h)
try {
    if (!h) return LAMA_OK;
    delete h->t;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
// setMaxDistance (:210-213)
int lama_tsdm_set_max_distance(lama_tsdm* h, double distance)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->t->set_max_distance(distance);
    return LAMA_OK;
}
LAMA_CATCH
// maxDistance (:215-218)
int lama_tsdm_max_distance(lama_tsdm* h, double* distance)
try {
    if (!h || !distance) return set_err("null argument", LAMA_ERR_ARG);
    *distance = h->t->max_distance();
    return LAMA_OK;
}
LAMA_CATCH
// insertPointCloud (:141-158), n_clouds of them in order
int lama_tsdm_insert_point_clouds(lama_tsdm* h, const double* pts_xyz, const int64_t* offsets, int n_clouds, const double* origins,
                                  const double* quats_xyzw, uint64_t* inserted)
try {
    if (!h || (n_clouds > 0 && !offsets)) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->t->insert_point_clouds(pts_xyz, offsets, n_clouds, origins, quats_xyzw, inserted);
    return rc == LAMA_OK ? rc : set_err(h->t->error(), rc);
}
LAMA_CATCH
// distance(Vector3d, gradient) (:59-130)
int lama_tsdm_distance(lama_tsdm* h, const double* pts_xyz, int n, double* distance, double* gradient)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    int rc = h->t->distance(pts_xyz, n, distance, gradient);
    return rc == LAMA_OK ? rc : set_err(h->t->error(), rc);
}
LAMA_CATCH
// Map::bounds (map.cpp:139-157)
int lama_tsdm_bounds(lama_tsdm* h, uint32_t mn[3], uint32_t mx[3], int* patches)
try {
    if (!h || !mn || !mx) return set_err("null argument", LAMA_ERR_ARG);
    return h->t->bounds(mn, mx, patches);
}
LAMA_CATCH
int lama_tsdm_export(lama_tsdm* h, const uint32_t lo[3], const int32_t size[3], float* distance, float* weight, uint8_t* on)
try {
    if (!h || !lo || !size) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->t->export_box(lo, size, distance, weight, on);
    return rc == LAMA_OK ? rc : set_err(h->t->error(), rc);
}
LAMA_CATCH
// toMesh (:220-272)
int lama_tsdm_to_mesh(lama_tsdm* h, float* vertices, size_t cap, size_t* n_vertices)
try {
    if (!h || !n_vertices) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->t->to_mesh(vertices, cap, n_vertices);
    return rc == LAMA_OK ? rc : set_err(h->t->error(), rc);
}
LAMA_CATCH
// sdm::export_to_ply (export.cpp:112-143)
int lama_tsdm_write_ply(lama_tsdm* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    size_t n = 0;
    int rc = h->t->to_mesh(nullptr, 0, &n);
    std::vector<float> v(n * 3);
    if (rc == LAMA_OK && n) rc = h->t->to_mesh(v.data(), n, &n);
    if (rc != LAMA_OK) return set_err(h->t->error(), rc);
    FILE* f = std::fopen(path, "w");
    if (!f) return set_err(std::string("cannot open file '") + path + "'", LAMA_ERR_ARG);
    std::fprintf(f, "ply\nformat ascii 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\nelement face %zu\n"
                    "property list uchar int vertex_index\nend_header\n", n, n / 3);
    for (size_t i = 0; i < n; ++i) std::fprintf(f, "%f %f %f\n", (double)v[3 * i], (double)v[3 * i + 1], (double)v[3 * i + 2]);
    for (size_t i = 0; i + 2 < n; i += 3) std::fprintf(f, "3 %d %d %d\n", (int)(i + 2), (int)(i + 1), (int)i);
    const bool ok = std::fclose(f) == 0;
    return ok ? LAMA_OK : set_err(std::string("cannot write file '") + path + "'", LAMA_ERR_ARG);
}
LAMA_CATCH
int lama_tsdm_kernel_times(lama_tsdm* h, double ms[3], uint64_t launches[3])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->t->kernel_times(ms, launches);
    return LAMA_OK;
}
LAMA_CATCH

// ---- 3-D occupancy maps (include/lama/sdm/frequency_occupancy_map.h, probabilistic_occupancy_map.h with is3d) ----------------------
struct lama_om3 { OccMap3Dev* m; };
// FrequencyOccupancyMap / ProbabilisticOccupancyMap(resolution, patch_size, true) (frequency_occupancy_map.cpp:47-49,
// probabilistic_occupancy_map.cpp:48-60, map.cpp:42-48) on the device
int lama_om3_create(double resolution, uint32_t patch_size, int kind, const double center_xyz[3], const int32_t window_patches[3],
                    const lama_device_options* dev, lama_om3** out)
try {
    if (!out) return set_err("null argument", LAMA_ERR_ARG);
    lama_device_options d;
    if (dev) d = *dev; else dev_default(&d);
    std::string err;
    OccMap3Dev* m = OccMap3Dev::create(resolution, patch_size, kind, center_xyz, window_patches, dev_from(d), err);
    if (!m) {
        const bool bad_arg = !(resolution > 0) || patch_size != 32 || (kind != 0 && kind != 1) || err.find("window") != std::string::npos;
        return set_err(err, !bad_arg && lama_b200::cuda_device_count() < 1 ? LAMA_ERR_NO_DEVICE : (bad_arg ? LAMA_ERR_ARG : LAMA_ERR_CUDA));
    }
    *out = new lama_om3{m};
    return LAMA_OK;
}
LAMA_CATCH
int lama_om3_destroy(lama_om3* h)
try {
    if (!h) return LAMA_OK;
    delete h->m;
    delete h;
    return LAMA_OK;
}
LAMA_CATCH
// the loop body of GraphSlam2D::generateOccupancyMap (graph_slam2d.cpp:146-158) over every point of every cloud
int lama_om3_insert_point_clouds(lama_om3* h, const double* pts_xyz, const int64_t* offsets, int n_clouds, const double* origins,
                                 const double* quats_xyzw, int full, uint64_t* cells)
try {
    if (!h || (n_clouds > 0 && !offsets)) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->m->insert_point_clouds(pts_xyz, offsets, n_clouds, origins, quats_xyzw, full != 0, cells);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// setFree / setOccupied / setUnknown (frequency_occupancy_map.cpp:65-108, probabilistic_occupancy_map.cpp:82-123) in list order
int lama_om3_apply(lama_om3* h, const uint32_t* cells_xyz, const uint8_t* ops, int n, uint8_t* changed)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    int rc = h->m->apply(cells_xyz, ops, n, changed);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// getProbability / isFree / isOccupied / isUnknown (frequency_occupancy_map.cpp:110-172, probabilistic_occupancy_map.cpp:125-175)
int lama_om3_query(lama_om3* h, const uint32_t* cells_xyz, int n, double* prob, uint8_t* flags)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    int rc = h->m->query(cells_xyz, n, prob, flags);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// FrequencyOccupancyMap::prune (frequency_occupancy_map.cpp:149-158)
int lama_om3_prune(lama_om3* h)
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    int rc = h->m->prune();
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// Map::bounds (map.cpp:139-157)
int lama_om3_bounds(lama_om3* h, uint32_t mn[3], uint32_t mx[3], int* patches)
try {
    if (!h || !mn || !mx) return set_err("null argument", LAMA_ERR_ARG);
    return h->m->bounds(mn, mx, patches);
}
LAMA_CATCH
// the cells of a box, as Map::get (map.cpp:414-455) reads them
int lama_om3_export(lama_om3* h, const uint32_t lo[3], const int32_t size[3], uint32_t* cells, uint8_t* known)
try {
    if (!h || !lo || !size) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->m->export_box(lo, size, cells, known);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// Map::write (map.cpp:490-529)
int lama_om3_write(lama_om3* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->m->write(path);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// Map::read (map.cpp:531-575)
int lama_om3_read(lama_om3* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->m->read(path);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
// sdm::export_to_png(occ, file, zed) (export.cpp:46-72,98-103): the grey image
int lama_om3_export_image(lama_om3* h, double zed, uint8_t* pixels, size_t cap, int dims[2])
try {
    if (!h || !dims) return set_err("null argument", LAMA_ERR_ARG);
    int rc = h->m->export_image(zed, pixels, cap, dims);
    return rc == LAMA_OK ? rc : set_err(h->m->error(), rc);
}
LAMA_CATCH
int lama_om3_kernel_times(lama_om3* h, double ms[3], uint64_t launches[3])
try {
    if (!h) return set_err("null handle", LAMA_ERR_ARG);
    h->m->kernel_times(ms, launches);
    return LAMA_OK;
}
LAMA_CATCH
// Map::w2m (map.h:125-126), all three axes
int lama_w2m3(double resolution, const double* pts_xyz, int n, uint32_t* cells_xyz)
try {
    if (!(resolution > 0) || n < 0 || (n > 0 && (!pts_xyz || !cells_xyz))) return set_err("bad argument", LAMA_ERR_ARG);
    const double scale = 1.0 / resolution;
    for (int i = 0; i < 3 * n; ++i) cells_xyz[i] = w2m(pts_xyz[i], scale);
    return LAMA_OK;
}
LAMA_CATCH

// ---- checkpoints (no counterpart in the reference) -----------------------------------------------------------
namespace {
thread_local CheckpointStats g_ckpt;
DeviceOptions load_dev(const lama_device_options* d)   // only device, stream and timing are taken; the geometry fields are checked
{
    DeviceOptions o;
    o.device = d ? d->device : 0;
    o.dir_dim = d ? d->dir_dim : 0;
    o.pool_slots = d ? d->pool_slots : 0;
    o.max_beams = d ? d->max_beams : 0;
    o.timing = d ? d->timing : 0;
    o.stream = d ? d->stream : 0;
    return o;
}
}  // namespace
int lama_pf_save_state(lama_pf* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    const int rc = h->p->save(path, &g_ckpt);
    return rc == LAMA_OK ? rc : set_err(h->p->error(), rc);
}
LAMA_CATCH
int lama_pf_load_state(const char* path, const lama_device_options* dev, lama_pf** out)
try {
    if (!path || !out) return set_err("null argument", LAMA_ERR_ARG);
    *out = nullptr;
    std::string err;
    int rc = LAMA_OK;
    PFSlam2D* p = PFSlam2D::load(path, load_dev(dev), err, &rc, &g_ckpt);
    if (!p) return set_err(err, rc == LAMA_OK ? LAMA_ERR_ARG : rc);
    *out = new lama_pf{p};
    return LAMA_OK;
}
LAMA_CATCH
int lama_slam_save_state(lama_slam* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    const int rc = h->s->save(path, &g_ckpt);
    return rc == LAMA_OK ? rc : set_err(h->s->error(), rc);
}
LAMA_CATCH
int lama_slam_load_state(const char* path, const lama_device_options* dev, lama_slam** out)
try {
    if (!path || !out) return set_err("null argument", LAMA_ERR_ARG);
    *out = nullptr;
    std::string err;
    int rc = LAMA_OK;
    Slam2D* s = Slam2D::load(path, load_dev(dev), err, &rc, &g_ckpt);
    if (!s) return set_err(err, rc == LAMA_OK ? LAMA_ERR_ARG : rc);
    *out = new lama_slam{s};
    return LAMA_OK;
}
LAMA_CATCH
int lama_graph_save_state(lama_graph* h, const char* path)
try {
    if (!h || !path) return set_err("null argument", LAMA_ERR_ARG);
    const int rc = h->g->save(path, &g_ckpt);
    return rc == LAMA_OK ? rc : set_err(h->g->error(), rc);
}
LAMA_CATCH
int lama_graph_load_state(const char* path, const lama_device_options* dev, lama_graph** out)
try {
    if (!path || !out) return set_err("null argument", LAMA_ERR_ARG);
    *out = nullptr;
    std::string err;
    int rc = LAMA_OK;
    GraphSlam2D* g = GraphSlam2D::load(path, load_dev(dev), err, &rc, &g_ckpt);
    if (!g) return set_err(err, rc == LAMA_OK ? LAMA_ERR_ARG : rc);
    *out = new lama_graph{g, lama_slam{g->slam(), false}, lama_om{g->occupancy_map(), false}, lama_dm{nullptr, false}};
    return LAMA_OK;
}
LAMA_CATCH
int lama_checkpoint_last_stats(double ms[9], uint64_t sizes[3])
try {
    if (!ms || !sizes) return set_err("null argument", LAMA_ERR_ARG);
    const CheckpointStats& s = g_ckpt;
    const double v[9] = {s.dev.count_ms, s.dev.compact_ms, s.dev.gather_ms, s.dev.copy_ms, s.dev.create_ms, s.dev.tables_ms, s.encode_ms, s.io_ms, s.total_ms};
    std::copy(v, v + 9, ms);
    sizes[0] = s.used_slots; sizes[1] = s.references; sizes[2] = s.file_bytes;
    return LAMA_OK;
}
LAMA_CATCH

}  // extern "C"
