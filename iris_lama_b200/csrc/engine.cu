// engine.cu -- device memory, stream and kernel pipeline behind the front ends.
#include "engine.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>

#include "kernels.cuh"

namespace lama_b200 {

#define CU_TRY(expr)                                                                                   \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(_e), LAMA_ERR_CUDA); \
    } while (0)

struct Engine::Impl {
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    StoreView view{};
    // scan
    double* d_points = nullptr;      // current scan (points into d_scan_buf or d_staged)
    double* d_scan_buf = nullptr;
    double* d_staged = nullptr;
    int staged_scans = 0, staged_beams = 0;
    ScanParams scan{};
    // per-launch staging
    SE2* d_states = nullptr;
    SE2* h_states = nullptr;  // pinned
    MatchResult* d_results = nullptr;
    MatchResult* h_results = nullptr;  // pinned
    MapUpdateStats* d_stats = nullptr;
    MapUpdateStats* h_stats = nullptr;  // pinned; two halves (ping-pong between consecutive map updates)
    uint64_t* h_report = nullptr;       // pinned; per half: {status, allocated, detached, freed, free slots}
    double* h_scan = nullptr;           // pinned staging of a host scan (step_async)
    cudaEvent_t ev_match = nullptr, ev_sync = nullptr;
    uint64_t* d_events = nullptr;
    int32_t* d_idx = nullptr;
    int32_t* h_idx = nullptr;  // pinned
    uint32_t* h_status = nullptr;  // pinned
    int state_cap = 0;
    RayParams ray{};
    BrushParams brush{};
    int n_sms = 132;
    int pull_max_particles = 0;   // the pull form of the ray cast is used up to this many particles per device; 0 = never (the walk is not slower at any
                                  // count, see launch_ray_stage); LAMA_PULL_MAX_PARTICLES overrides
    bool scan_flat = false;     // the current scan has z == 0 everywhere and a sensor that keeps z planes: every beam is planar
    bool staged_flat = false;   // the same for the staged scans
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    // timing of the pipelined step (step_enqueue): per report buffer {before match, after match, after the ray stage, after the brushfire}; read when
    // that step is collected, so no host synchronisation is added
    cudaEvent_t evp[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};
    bool evp_used[2] = {false, false};
    // scratch for import/export/distance
    void* d_scratch = nullptr;
    size_t scratch_bytes = 0;
    // device arena of a migration round (pack_device / migration_alloc): bump allocation out of chunks that are kept between rounds, so that a resampling
    // scan costs no cudaMalloc / cudaFree once the arena has grown to its working size
    std::vector<std::pair<char*, size_t>> mig_chunks;
    size_t mig_chunk = 0, mig_off = 0;
    std::vector<void*> allocs;
};


constexpr int kPullMaxBeams = 4096;   // k_ray_setup sorts the beams of a scan in shared memory

static bool points_flat(const double* pts, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        if (pts[3 * i + 2] != 0.0) return false;
    return true;
}

// The occupancy ray cast of `count` particles.  Scans whose beams all start in the same cell (no per-beam ray truncation) go through
// the pull form (k_ray_setup + k_ray_pull); k_raycast, the per-beam walk, takes everything else: LidarOdometry2D's and truncated rays,
// and -- decided per particle on the device -- scans of a tilted sensor (`flat` false: the beams may leave the z plane).
static int launch_ray_stage(Engine::Impl* d, RayParams rp, const SE2* states, int count)   // returns the number of kernels launched
{
    const ScanParams& sp = rp.scan;
    // The walk runs one CTA per particle, the pull form spreads the patches of all particles over every SM.  Measured on an H100 (scripts/pull_variants.py,
    // revisit regime): walk 0.152 / 0.200 / 0.318 / 0.636 ms, pull 0.227 / 0.287 / 0.393 / 0.632 ms at 32 / 64 / 128 / 256 particles -- the walk wins
    // up to 128 and ties at 256, so pull_max_particles defaults to 0; LAMA_PULL_MAX_PARTICLES (read when the engine is created) selects the pull
    // form up to that many particles per device.
    const bool no_pull = count > d->pull_max_particles;
    const bool flat = d->scan_flat && sp.moving.l[6] == 0.0 && sp.moving.l[7] == 0.0;
    rp.pull_fallback = 0;
    if (!no_pull && !sp.lo_ray && sp.truncated_ray == 0.0 && sp.n_beams <= kPullMaxBeams) {
        launch_raycast_pull(d->view, rp, states, d->d_events, d->d_stats, count, d->n_sms, d->stream);
        if (flat) return 2;   // hit.z == start.z exactly for every beam: k_ray_setup takes every particle
        rp.pull_fallback = 1;
    }
    launch_raycast(d->view, rp, states, d->d_events, d->d_stats, count, d->stream);
    return rp.pull_fallback ? 3 : 1;
}

int cuda_device_count()
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int Engine::fail(const std::string& what, int code)
{
    err_ = what;
    return code;
}

static int next_pow2_host(int v)
{
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

Engine* Engine::create(const EngineConfig& cfg, std::string& err)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        err = "no CUDA device available: the lama_b200 hot path has no CPU fallback";
        return nullptr;
    }
    if (cfg.device < 0 || cfg.device >= ndev) {
        err = "invalid device index";
        return nullptr;
    }
    if (cfg.particles < 1 || cfg.dir_dim < 8 || cfg.dir_dim > 128 || (cfg.dir_dim & (cfg.dir_dim - 1)) != 0 || cfg.max_beams < 1 ||
        cfg.max_beams > 32768 || !(cfg.resolution > 0)) {
        err = "invalid engine configuration (particles >= 1, dir_dim power of two in [8,128], max_beams <= 32768)";
        return nullptr;
    }
    const double scale = 1.0 / cfg.resolution;
    uint32_t radius = (uint32_t)std::ceil(cfg.l2_max * scale);  // DynamicDistanceMap::setMaxDistance, dynamic_distance_map.cpp:149-153
    if (radius > (uint32_t)kDmMaxRadius) {
        err = "l2_max * scale exceeds 63 cells (packed distance cell limit)";
        return nullptr;
    }
    Engine* e = new Engine();
    e->cfg_ = cfg;
    e->max_sqdist_ = radius * radius;
    if (e->cfg_.pool_slots <= 0) {
        const long long want = (long long)cfg.particles * 768 + 1024;
        e->cfg_.pool_slots = want >= (long long)kDirSlotMask ? kDirSlotMask - 1 : (int)want;
    }
    if (e->cfg_.pool_slots >= kDirSlotMask) {   // directory entries keep the slot in 24 bits, all ones = "not writable"
        err = "pool_slots must be below 2^24 - 1 (the slot field of a directory entry)";
        delete e;
        return nullptr;
    }
    Impl* d = e->d_ = new Impl();
    auto bail = [&](const std::string& m) {
        err = m;
        delete e;
        return (Engine*)nullptr;
    };
#define CU_NEW(expr)                                                             \
    do {                                                                         \
        cudaError_t _e = (expr);                                                 \
        if (_e != cudaSuccess) return bail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
    CU_NEW(cudaSetDevice(cfg.device));
    if (cfg.stream) {
        d->stream = reinterpret_cast<cudaStream_t>(cfg.stream);
        d->own_stream = false;
    } else {
        CU_NEW(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
    }
    CU_NEW(cudaEventCreate(&d->ev[0]));
    CU_NEW(cudaEventCreate(&d->ev[1]));
    CU_NEW(cudaEventCreate(&d->ev[2]));
    for (int b = 0; b < 2; ++b)
        for (int k = 0; k < 4; ++k) CU_NEW(cudaEventCreate(&d->evp[b][k]));

    // directory window centred on (center_x, center_y)
    const uint32_t cx = w2m(cfg.center_x, scale), cy = w2m(cfg.center_y, scale);
    e->window_.dim     = cfg.dir_dim;
    e->window_.base_px = (int32_t)(cx >> kPatchLog2) - cfg.dir_dim / 2;
    e->window_.base_py = (int32_t)(cy >> kPatchLog2) - cfg.dir_dim / 2;

    StoreView& v = d->view;
    v.n_slots     = e->cfg_.pool_slots;
    v.n_particles = cfg.particles;
    v.n_kinds     = cfg.occupancy_kind == 1 ? 3 : 2;
    v.kbits       = nullptr;
    v.window      = e->window_;
    const size_t dim2 = (size_t)cfg.dir_dim * cfg.dir_dim;
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t r = cudaMalloc(p, bytes);
        if (r == cudaSuccess) d->allocs.push_back(*p);
        return r;
    };
    // k_raycast ORs cell offsets into patch base addresses: the pool starts on a 4 KiB boundary (cudaMalloc only promises 256 B)
    CU_NEW(dalloc((void**)&v.pool, ((size_t)v.n_slots + 1) * kPatchBytes));
    v.pool = reinterpret_cast<uint32_t*>(((uintptr_t)v.pool + (kPatchBytes - 1)) & ~(uintptr_t)(kPatchBytes - 1));
    CU_NEW(dalloc((void**)&v.fbits, (size_t)v.n_slots * 128));
    if (cfg.occupancy_kind == 1 || cfg.known_plane) CU_NEW(dalloc((void**)&v.kbits, (size_t)v.n_slots * 128));
    CU_NEW(dalloc((void**)&v.refcount, (size_t)v.n_slots * 4));
    CU_NEW(dalloc((void**)&v.free_slots, (size_t)v.n_slots * 4));
    CU_NEW(dalloc((void**)&v.freed, (size_t)v.n_slots * 4));
    CU_NEW(dalloc((void**)&v.free_count, 64));
    v.freed_count = v.free_count + 1;
    v.status      = reinterpret_cast<uint32_t*>(v.free_count + 2);
    v.counters    = reinterpret_cast<uint64_t*>(v.free_count + 4);
    CU_NEW(dalloc((void**)&v.dirs, 2 * (size_t)cfg.particles * v.n_kinds * dim2 * 4));
    CU_NEW(dalloc((void**)&d->d_scan_buf, (size_t)cfg.max_beams * 3 * 8));
    d->d_points = d->d_scan_buf;

    d->ray.log_cap   = next_pow2_host(std::max(4096, 3 * cfg.max_beams));
    d->ray.cand_cap  = 192;
    if (const char* cc = std::getenv("LAMA_RAY_CAND_CAP")) {   // test hook: force the candidate-overflow path of k_raycast
        const int v = std::atoi(cc);
        d->ray.cand_cap = v < 1 ? 1 : (v > 253 ? 253 : v);
    }
    d->ray.prob_mode = cfg.occupancy_kind == 1 ? 1 : 0;
    {   // ProbabilisticOccupancyMap's constructor (probabilistic_occupancy_map.cpp:43-60): float logods(), stored as doubles
        auto logods = [](float prob) -> float { return (float)std::log(prob / (1.0 - prob)); };
        d->ray.prob.miss      = logods(0.4f);
        d->ray.prob.hit       = logods(0.7f);
        d->ray.prob.clamp_min = logods(0.12f);
        d->ray.prob.clamp_max = logods(0.97f);
        d->ray.prob.thresh    = 0.0 * logods(0.5f);
    }
    d->ray.event_cap = next_pow2_host(std::max(std::max(2048, cfg.max_beams), cfg.event_cap));
    d->ray.scan.n_beams = cfg.max_beams;  // shared-memory budget is registered for the largest scan
    d->brush.event_cap = d->ray.event_cap;
    d->brush.lower_cap = 8192;
    d->brush.raise_cap = 2048;
    d->brush.max_sqdist = e->max_sqdist_;
    CU_NEW(dalloc((void**)&d->d_events, (size_t)cfg.particles * d->ray.event_cap * 8));
    {   // scratch of the pull ray cast (k_ray_setup -> k_ray_pull)
        RayPullView& pv = d->ray.pull;
        pv.stride = (std::min(cfg.max_beams, kPullMaxBeams) + 31) & ~31;
        if (pv.stride < 32) pv.stride = 32;
        int npad = 32;
        while (npad < pv.stride) npad <<= 1;
        pv.stride = npad;   // k_ray_setup writes whole sorted arrays of next_pow2(beams) entries
        CU_NEW(dalloc((void**)&pv.hdr, (size_t)cfg.particles * sizeof(RayPullHeader)));
        CU_NEW(dalloc((void**)&pv.list, (size_t)cfg.particles * pv.stride * sizeof(PullEntry)));
        CU_NEW(dalloc((void**)&pv.hits, (size_t)cfg.particles * pv.stride * 4));
        CU_NEW(dalloc((void**)&pv.tasks, (size_t)cfg.particles * dim2 * 8));
        CU_NEW(dalloc((void**)&pv.ctrl, 64));
        CU_NEW(cudaMemset(pv.ctrl, 0, 64));
        CU_NEW(cudaMemset(pv.hdr, 0, (size_t)cfg.particles * sizeof(RayPullHeader)));
        v.ray_ctrl = pv.ctrl;
        int sms = 0;
        CU_NEW(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg.device));
        d->n_sms = sms > 0 ? sms : 132;
        if (const char* pm = std::getenv("LAMA_PULL_MAX_PARTICLES")) d->pull_max_particles = std::atoi(pm);
    }
    CU_NEW(dalloc((void**)&d->d_stats, (size_t)cfg.particles * sizeof(MapUpdateStats)));
    const size_t idx_ints = std::max((size_t)cfg.particles, (size_t)cfg.dir_dim * cfg.dir_dim);   // resample indices / directory entries to delete
    CU_NEW(dalloc((void**)&d->d_idx, idx_ints * 4));
    CU_NEW(cudaMallocHost((void**)&d->h_stats, 2 * (size_t)cfg.particles * sizeof(MapUpdateStats)));
    CU_NEW(cudaMallocHost((void**)&d->h_report, 2 * 8 * sizeof(uint64_t)));
    std::memset(d->h_report, 0, 2 * 8 * sizeof(uint64_t));
    CU_NEW(cudaMallocHost((void**)&d->h_scan, (size_t)cfg.max_beams * 24));
    CU_NEW(cudaEventCreateWithFlags(&d->ev_match, cudaEventDisableTiming));
    CU_NEW(cudaEventCreateWithFlags(&d->ev_sync, cudaEventDisableTiming));
    CU_NEW(cudaMallocHost((void**)&d->h_idx, idx_ints * 4));
    CU_NEW(cudaMallocHost((void**)&d->h_status, 64));

    const size_t need_ray = raycast_smem_bytes(cfg.dir_dim, d->ray), need_match = match_smem_bytes(cfg.dir_dim, e->max_sqdist_),
                 need_brush = brushfire_smem_bytes(cfg.dir_dim, d->brush);
    if (need_ray > 227 * 1024 || need_match > 227 * 1024 || need_brush > 227 * 1024) return bail("shared memory budget exceeded (reduce max_beams / dir_dim)");
    CU_NEW(configure_kernels(cfg.dir_dim, e->max_sqdist_, d->ray, d->brush));

    launch_init_store(v, 2, d->stream);
    CU_NEW(cudaGetLastError());
    CU_NEW(cudaStreamSynchronize(d->stream));
#undef CU_NEW
    return e;
}

Engine::~Engine()
{
    if (!d_) return;
    cudaSetDevice(cfg_.device);
    if (d_->stream) cudaStreamSynchronize(d_->stream);
    for (void* p : d_->allocs) cudaFree(p);
    if (d_->d_states) cudaFree(d_->d_states);
    if (d_->d_results) cudaFree(d_->d_results);
    if (d_->h_states) cudaFreeHost(d_->h_states);
    if (d_->h_results) cudaFreeHost(d_->h_results);
    if (d_->h_stats) cudaFreeHost(d_->h_stats);
    if (d_->h_report) cudaFreeHost(d_->h_report);
    if (d_->h_scan) cudaFreeHost(d_->h_scan);
    if (d_->ev_match) cudaEventDestroy(d_->ev_match);
    if (d_->ev_sync) cudaEventDestroy(d_->ev_sync);
    for (auto& c : d_->mig_chunks) cudaFree(c.first);
    if (d_->h_idx) cudaFreeHost(d_->h_idx);
    if (d_->h_status) cudaFreeHost(d_->h_status);
    if (d_->d_scratch) cudaFree(d_->d_scratch);
    if (d_->d_staged) cudaFree(d_->d_staged);
    for (int b = 0; b < 2; ++b)
        for (int k = 0; k < 4; ++k)
            if (d_->evp[b][k]) cudaEventDestroy(d_->evp[b][k]);
    if (d_->ev[0]) cudaEventDestroy(d_->ev[0]);
    if (d_->ev[1]) cudaEventDestroy(d_->ev[1]);
    if (d_->ev[2]) cudaEventDestroy(d_->ev[2]);
    if (d_->stream && d_->own_stream) cudaStreamDestroy(d_->stream);
    delete d_;
}

int Engine::synchronize()
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    CU_TRY(cudaSetDevice(cfg_.device));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    return LAMA_OK;
}

// Translation3d(sensor_origin) * Quaterniond  (match_surface_2d.cpp:49; Eigen quaternion -> matrix); null = identity
MovingTf moving_tf(const double origin[3], const double quat[4])
{
    MovingTf m;
    const double x = quat ? quat[0] : 0, y = quat ? quat[1] : 0, z = quat ? quat[2] : 0, w = quat ? quat[3] : 1;
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    double* l = m.l;
    l[0] = 1 - (tyy + tzz); l[1] = txy - twz;       l[2] = txz + twy;
    l[3] = txy + twz;       l[4] = 1 - (txx + tzz); l[5] = tyz - twx;
    l[6] = txz - twy;       l[7] = tyz + twx;       l[8] = 1 - (txx + tyy);
    for (int i = 0; i < 3; ++i) m.t[i] = origin ? origin[i] : 0.0;
    return m;
}

void Engine::set_moving(const double origin[3], const double quat[4], double truncated_ray, double truncated_range, int n)
{
    ScanParams& sp = d_->scan;
    sp.n_beams         = n;
    sp.scale           = 1.0 / cfg_.resolution;
    sp.truncated_ray   = truncated_ray;
    sp.truncated_range = truncated_range;
    sp.lo_ray          = lo_ray_ ? 1 : 0;
    sp.moving          = moving_tf(origin, quat);
}

int Engine::set_scan(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (!pts || n < 1 || n > cfg_.max_beams) return fail("set_scan: number of beams out of range", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    set_moving(origin, quat, truncated_ray, truncated_range, n);
    d_->d_points = d_->d_scan_buf;
    d_->scan_flat = points_flat(pts, (size_t)n);
    // pageable host memory: cudaMemcpyAsync stages through the driver; the copy is small (N * 24 B)
    CU_TRY(cudaMemcpyAsync(d_->d_points, pts, (size_t)n * 3 * 8, cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));  // `pts` may be released by the caller after return
    h2d_bytes_ += (uint64_t)n * 24;
    return LAMA_OK;
}

int Engine::stage_scans(const double* pts, int n_scans, int n)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (!pts || n_scans < 1 || n < 1 || n > cfg_.max_beams) return fail("stage_scans: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    if (d_->d_staged) { cudaFree(d_->d_staged); d_->d_staged = nullptr; }
    CU_TRY(cudaMalloc((void**)&d_->d_staged, (size_t)n_scans * n * 24));
    CU_TRY(cudaMemcpyAsync(d_->d_staged, pts, (size_t)n_scans * n * 24, cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    d_->staged_scans = n_scans;
    d_->staged_beams = n;
    d_->staged_flat  = points_flat(pts, (size_t)n_scans * n);
    return LAMA_OK;
}

int Engine::select_staged(int index, const double origin[3], const double quat[4], double truncated_ray, double truncated_range)
{
    if (!d_->d_staged || index < 0 || index >= d_->staged_scans) return fail("select_staged: no such staged scan", LAMA_ERR_ARG);
    set_moving(origin, quat, truncated_ray, truncated_range, d_->staged_beams);
    d_->d_points = d_->d_staged + (size_t)index * d_->staged_beams * 3;
    d_->scan_flat = d_->staged_flat;
    return LAMA_OK;
}

int Engine::ensure_states(int count)
{
    if (count <= d_->state_cap) return LAMA_OK;
    if (d_->d_states) { cudaFree(d_->d_states); cudaFree(d_->d_results); cudaFreeHost(d_->h_states); cudaFreeHost(d_->h_results); }
    d_->d_states = nullptr; d_->d_results = nullptr; d_->h_states = nullptr; d_->h_results = nullptr;
    d_->state_cap = 0;
    const int cap = std::max(count, cfg_.particles);
    CU_TRY(cudaMalloc((void**)&d_->d_states, (size_t)cap * sizeof(SE2)));
    CU_TRY(cudaMalloc((void**)&d_->d_results, (size_t)cap * sizeof(MatchResult)));
    CU_TRY(cudaMallocHost((void**)&d_->h_states, (size_t)cap * sizeof(SE2)));
    CU_TRY(cudaMallocHost((void**)&d_->h_results, (size_t)cap * sizeof(MatchResult)));
    d_->state_cap = cap;
    return LAMA_OK;
}

int Engine::check_device_status()
{
    uint32_t st = *d_->h_status;
    if (!st) return LAMA_OK;
    if (st & kErrWindow) return fail("map grew outside the directory window (raise dir_dim)", LAMA_ERR_WINDOW);
    if (st & kErrPoolEmpty) return fail("patch pool exhausted (raise pool_slots)", LAMA_ERR_POOL);
    return fail("event log / heap overflow in the map update kernels", LAMA_ERR_OVERFLOW);
}

uint32_t Engine::device_status()
{
    settle(nullptr);
    cudaSetDevice(cfg_.device);
    cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream);
    cudaStreamSynchronize(d_->stream);
    return *d_->h_status;
}

void Engine::store_counters(uint64_t out[4])
{
    settle(nullptr);
    cudaSetDevice(cfg_.device);
    uint64_t c[3];
    int32_t fc = 0;
    cudaMemcpyAsync(c, d_->view.counters, sizeof(c), cudaMemcpyDeviceToHost, d_->stream);
    cudaMemcpyAsync(&fc, d_->view.free_count, 4, cudaMemcpyDeviceToHost, d_->stream);
    cudaStreamSynchronize(d_->stream);
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = (uint64_t)fc;
}

int Engine::match(const SE2* states, int count, int first_particle, bool shared_map, const SolverOptions& so, double meas_sigma, int mode,
                  HostMatchResult* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count < 1 || first_particle < 0 || (!shared_map && first_particle + count > cfg_.particles) || first_particle >= cfg_.particles)
        return fail("match: particle range out of bounds", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("match: no scan uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = ensure_states(count); if (rc != LAMA_OK) return rc; }
    std::memcpy(d_->h_states, states, (size_t)count * sizeof(SE2));
    CU_TRY(cudaMemcpyAsync(d_->d_states, d_->h_states, (size_t)count * sizeof(SE2), cudaMemcpyHostToDevice, d_->stream));
    MatchParams mp{};
    mp.points = d_->d_points;
    mp.scan = d_->scan;
    mp.solver = so;
    mp.meas_sigma = meas_sigma;
    mp.resolution = cfg_.resolution;
    mp.max_sqdist = max_sqdist_;
    mp.set = cur_set_;
    mp.particle_offset = first_particle;
    mp.shared_map = shared_map ? 1 : 0;
    mp.mode = mode;
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    launch_match(d_->view, mp, d_->d_states, d_->d_results, count, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_results, d_->d_results, (size_t)count * sizeof(MatchResult), cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_) {
        float ms = 0;
        cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]);
        times_.match_ms += ms;
    }
    times_.match_launches += 1;
    static_assert(sizeof(HostMatchResult) == sizeof(MatchResult), "layout");
    std::memcpy(out, d_->h_results, (size_t)count * sizeof(MatchResult));
    h2d_bytes_ += (uint64_t)count * sizeof(SE2);
    d2h_bytes_ += (uint64_t)count * sizeof(MatchResult);
    return LAMA_OK;
}

int Engine::match_error(const SE2* states, int count, int first_particle, bool shared_map, double* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count < 1 || first_particle < 0 || (!shared_map && first_particle + count > cfg_.particles) || first_particle >= cfg_.particles)
        return fail("match_error: particle range out of bounds", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("match_error: no scan uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = ensure_states(count); if (rc != LAMA_OK) return rc; }
    std::memcpy(d_->h_states, states, (size_t)count * sizeof(SE2));
    CU_TRY(cudaMemcpyAsync(d_->d_states, d_->h_states, (size_t)count * sizeof(SE2), cudaMemcpyHostToDevice, d_->stream));
    double* d_out = reinterpret_cast<double*>(d_->d_results);   // count doubles fit in count MatchResults
    launch_match_error(d_->view, cur_set_, first_particle, shared_map, d_->d_points, d_->scan, d_->d_states, count, cfg_.resolution, max_sqdist_, d_out, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, d_out, (size_t)count * 8, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::update_maps(const SE2* states, int first_particle, int count, HostMapStats* out)
{
    int rc = update_maps_async(states, first_particle, count);
    if (rc != LAMA_OK) return rc;
    return settle(out);
}

// developer builds (LAMA_PHASE_TIMING): LAMA_BF_DEBUG = ordinal of the map update whose k_brushfire prints its per-particle phase cycles
static int brush_debug_flag()
{
    static int launch_no = 0;
    const char* dbg = std::getenv("LAMA_BF_DEBUG");
    return dbg && std::atoi(dbg) == launch_no++;
}

// Launches ray cast + brushfire and returns without waiting; settle() (called by every later entry point)
// synchronises, collects the per-particle statistics and surfaces device errors.
int Engine::update_maps_async(const SE2* states, int first_particle, int count)
{
    if (count < 1 || first_particle < 0 || first_particle + count > cfg_.particles) return fail("update_maps: particle range out of bounds", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("update_maps: no scan uploaded", LAMA_ERR_STATE);
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = ensure_states(count); if (rc != LAMA_OK) return rc; }
    std::memcpy(d_->h_states, states, (size_t)count * sizeof(SE2));
    CU_TRY(cudaMemcpyAsync(d_->d_states, d_->h_states, (size_t)count * sizeof(SE2), cudaMemcpyHostToDevice, d_->stream));
    RayParams rp = d_->ray;
    rp.points = d_->d_points;
    rp.scan = d_->scan;
    rp.set = cur_set_;
    rp.particle_offset = first_particle;
    rp.state_stride = (int)sizeof(SE2);
    { const char* dbg = std::getenv("LAMA_RAY_DEBUG"); rp.debug = dbg ? std::atoi(dbg) : 0; }  // see RayParams::debug
    // shared-memory scratch sized for THIS scan (two CTAs per SM at 1080 beams); the maxima were registered at create
    const int nb = d_->scan.n_beams;
    rp.log_cap   = std::min(d_->ray.log_cap, next_pow2_host(std::max(1024, 3 * nb)));
    rp.event_cap = std::min(d_->ray.event_cap, next_pow2_host(std::max(512, nb)));
    BrushParams bp = d_->brush;
    bp.set = cur_set_;
    bp.particle_offset = first_particle;
    bp.event_cap = rp.event_cap;
    bp.debug = brush_debug_flag();
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    const int ray_kernels = launch_ray_stage(d_, rp, d_->d_states, count);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    launch_brushfire(d_->view, bp, d_->d_events, d_->d_stats, count, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[2], d_->stream));
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    { int rc = enqueue_report(count); if (rc != LAMA_OK) return rc; }
    times_.raycast_launches += ray_kernels;
    times_.brushfire_launches += 1;
    times_.misc_launches += 1;
    h2d_bytes_ += (uint64_t)count * sizeof(SE2);
    return LAMA_OK;
}

// device -> host report of a map update into the other half of the ping-pong buffers (the previous half may not have been read yet)
int Engine::enqueue_report(int count)
{
    const int half = 1 - pending_buf_;
    MapUpdateStats* hs = d_->h_stats + (size_t)half * cfg_.particles;
    uint64_t* hr = d_->h_report + (size_t)half * 8;
    CU_TRY(cudaMemcpyAsync(hs, d_->d_stats, (size_t)count * sizeof(MapUpdateStats), cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(hr, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(hr + 1, d_->view.counters, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(hr + 4, d_->view.free_count, 4, cudaMemcpyDeviceToHost, d_->stream));
    d2h_bytes_ += (uint64_t)count * sizeof(MapUpdateStats) + 4 + 28;
    pending_buf_  = half;
    pending_maps_ = count;
    return LAMA_OK;
}

int Engine::step_enqueue(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                         const SE2* predicted, int count, const SolverOptions& so, double meas_sigma)
{
    if (count < 1 || count > cfg_.particles) return fail("step_enqueue: particle range out of bounds", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    // the previous scan's map update may still be running: nothing below waits for it on the host
    enq_had_pending_ = pending_maps_ != 0;
    enq_prev_count_  = pending_maps_;
    enq_prev_buf_    = pending_buf_;
    if (pts) {
        if (n < 1 || n > cfg_.max_beams) return fail("step_enqueue: number of beams out of range", LAMA_ERR_ARG);
        set_moving(origin, quat, truncated_ray, truncated_range, n);
        std::memcpy(d_->h_scan, pts, (size_t)n * 24);   // free again: the previous call returned after its match, which follows its upload
        d_->d_points = d_->d_scan_buf;
        d_->scan_flat = points_flat(pts, (size_t)n);
        CU_TRY(cudaMemcpyAsync(d_->d_points, d_->h_scan, (size_t)n * 24, cudaMemcpyHostToDevice, d_->stream));
        h2d_bytes_ += (uint64_t)n * 24;
    }
    if (d_->scan.n_beams < 1) return fail("step_enqueue: no scan selected", LAMA_ERR_STATE);
    { int rc = ensure_states(count); if (rc != LAMA_OK) return rc; }
    std::memcpy(d_->h_states, predicted, (size_t)count * sizeof(SE2));
    CU_TRY(cudaMemcpyAsync(d_->d_states, d_->h_states, (size_t)count * sizeof(SE2), cudaMemcpyHostToDevice, d_->stream));
    MatchParams mp{};
    mp.points = d_->d_points;
    mp.scan = d_->scan;
    mp.solver = so;
    mp.meas_sigma = meas_sigma;
    mp.resolution = cfg_.resolution;
    mp.max_sqdist = max_sqdist_;
    mp.set = cur_set_;
    mp.particle_offset = 0;
    mp.shared_map = 0;
    mp.mode = 0;
    const int tbuf = 1 - pending_buf_;   // the report buffer enqueue_report() will hand to this step
    if (timing_) CU_TRY(cudaEventRecord(d_->evp[tbuf][0], d_->stream));
    launch_match(d_->view, mp, d_->d_states, d_->d_results, count, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->evp[tbuf][1], d_->stream));
    CU_TRY(cudaMemcpyAsync(d_->h_results, d_->d_results, (size_t)count * sizeof(MatchResult), cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaEventRecord(d_->ev_match, d_->stream));
    // map update on the matched poses, read from the match results on the device
    RayParams rp = d_->ray;
    rp.points = d_->d_points;
    rp.scan = d_->scan;
    rp.set = cur_set_;
    rp.particle_offset = 0;
    rp.state_stride = (int)sizeof(MatchResult);
    const int nb = d_->scan.n_beams;
    rp.log_cap   = std::min(d_->ray.log_cap, next_pow2_host(std::max(1024, 3 * nb)));
    rp.event_cap = std::min(d_->ray.event_cap, next_pow2_host(std::max(512, nb)));
    BrushParams bp = d_->brush;
    bp.set = cur_set_;
    bp.particle_offset = 0;
    bp.event_cap = rp.event_cap;
    bp.debug = brush_debug_flag();
    const int ray_kernels = launch_ray_stage(d_, rp, reinterpret_cast<const SE2*>(d_->d_results), count);
    if (timing_) CU_TRY(cudaEventRecord(d_->evp[tbuf][2], d_->stream));
    launch_brushfire(d_->view, bp, d_->d_events, d_->d_stats, count, d_->stream);
    if (timing_) {
        CU_TRY(cudaEventRecord(d_->evp[tbuf][3], d_->stream));
        d_->evp_used[tbuf] = true;
    }
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    { int rc = enqueue_report(count); if (rc != LAMA_OK) return rc; }
    times_.match_launches += 1;
    times_.raycast_launches += ray_kernels;
    times_.brushfire_launches += 1;
    times_.misc_launches += 1;
    h2d_bytes_ += (uint64_t)count * sizeof(SE2);
    d2h_bytes_ += (uint64_t)count * sizeof(MatchResult);
    return LAMA_OK;
}

int Engine::collect_previous()
{
    // everything enqueued before this scan's match has completed: collect the previous map update without waiting
    if (!enq_had_pending_) return LAMA_OK;
    enq_had_pending_ = false;
    const int cur_count = pending_maps_, cur_buf = pending_buf_;
    pending_maps_ = enq_prev_count_;
    pending_buf_  = enq_prev_buf_;
    const int rc = settle(nullptr, true);
    pending_maps_ = cur_count;
    pending_buf_  = cur_buf;
    return rc;
}

int Engine::step_async(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                       const SE2* predicted, int count, const SolverOptions& so, double meas_sigma, HostMatchResult* out)
{
    { int rc = step_enqueue(pts, n, origin, quat, truncated_ray, truncated_range, predicted, count, so, meas_sigma); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaEventSynchronize(d_->ev_match));
    static_assert(sizeof(HostMatchResult) == sizeof(MatchResult), "layout");
    std::memcpy(out, d_->h_results, (size_t)count * sizeof(MatchResult));
    return collect_previous();
}

void* Engine::stream_handle() const { return d_->stream; }

int Engine::wait_for_stream(void* other_stream)
{
    CU_TRY(cudaSetDevice(cfg_.device));
    CU_TRY(cudaEventRecord(d_->ev_sync, d_->stream));
    CU_TRY(cudaStreamWaitEvent(reinterpret_cast<cudaStream_t>(other_stream), d_->ev_sync, 0));
    return LAMA_OK;
}

int Engine::pack_results(int count, double digest, double* d_out, void* stream)
{
    CU_TRY(cudaSetDevice(cfg_.device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CU_TRY(cudaStreamWaitEvent(st, d_->ev_match, 0));
    launch_pack_results(d_->d_results, count, digest, d_out, st);
    CU_TRY(cudaGetLastError());
    return LAMA_OK;
}

int Engine::settle(HostMapStats* out, bool already_complete)
{
    if (pending_maps_ == 0) return LAMA_OK;
    const int count = pending_maps_;
    pending_maps_ = 0;
    CU_TRY(cudaSetDevice(cfg_.device));
    if (!already_complete) CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_ && d_->evp_used[pending_buf_]) {   // a pipelined step: its four events have completed (the stream is past them, or was just synchronised)
        float m = 0, a = 0, b = 0;
        cudaEventElapsedTime(&m, d_->evp[pending_buf_][0], d_->evp[pending_buf_][1]);
        cudaEventElapsedTime(&a, d_->evp[pending_buf_][1], d_->evp[pending_buf_][2]);
        cudaEventElapsedTime(&b, d_->evp[pending_buf_][2], d_->evp[pending_buf_][3]);
        times_.match_ms += m;
        times_.raycast_ms += a;
        times_.brushfire_ms += b;
        d_->evp_used[pending_buf_] = false;
    } else if (timing_ && !already_complete) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, d_->ev[0], d_->ev[1]);
        cudaEventElapsedTime(&b, d_->ev[1], d_->ev[2]);
        times_.raycast_ms += a;
        times_.brushfire_ms += b;
    }
    static_assert(sizeof(HostMapStats) == sizeof(MapUpdateStats), "layout");
    const MapUpdateStats* hs = d_->h_stats + (size_t)pending_buf_ * cfg_.particles;
    const uint64_t* hr = d_->h_report + (size_t)pending_buf_ * 8;
    last_map_stats_.assign((const HostMapStats*)hs, (const HostMapStats*)hs + count);
    if (out) std::memcpy(out, hs, (size_t)count * sizeof(MapUpdateStats));
    settled_counters_[0] = hr[1]; settled_counters_[1] = hr[2]; settled_counters_[2] = hr[3];
    settled_counters_[3] = (uint64_t)(uint32_t)hr[4];
    *d_->h_status = (uint32_t)hr[0];
    return check_device_status();
}

int Engine::share_from(int src_particle, int dst_first, int count)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count == 0) return LAMA_OK;
    if (src_particle < 0 || src_particle >= cfg_.particles || dst_first < 0 || dst_first + count > cfg_.particles ||
        (src_particle >= dst_first && src_particle < dst_first + count))
        return fail("share_from: bad particle range", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    for (int i = 0; i < count; ++i) d_->h_idx[i] = src_particle;
    CU_TRY(cudaMemcpyAsync(d_->d_idx, d_->h_idx, (size_t)count * 4, cudaMemcpyHostToDevice, d_->stream));
    launch_release(d_->view, cur_set_, dst_first, count, d_->stream);
    launch_copy_dirs(d_->view, cur_set_, cur_set_, d_->d_idx, dst_first, count, d_->stream);
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 3;
    return LAMA_OK;
}

int Engine::resample(const int32_t* idx)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    CU_TRY(cudaSetDevice(cfg_.device));
    const int P = cfg_.particles;
    for (int i = 0; i < P; ++i) {
        if (idx[i] < -1 || idx[i] >= P) return fail("resample: index out of range", LAMA_ERR_ARG);
        d_->h_idx[i] = idx[i];
    }
    CU_TRY(cudaMemcpyAsync(d_->d_idx, d_->h_idx, (size_t)P * 4, cudaMemcpyHostToDevice, d_->stream));
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    const int other = 1 - cur_set_;
    launch_copy_dirs(d_->view, cur_set_, other, d_->d_idx, 0, P, d_->stream);  // share first ...
    launch_release(d_->view, cur_set_, 0, P, d_->stream);                       // ... then drop the old set
    launch_merge_free(d_->view, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_) {
        float ms = 0;
        cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]);
        times_.resample_ms += ms;
    }
    times_.resample_launches += 3;
    cur_set_ = other;
    return LAMA_OK;
}

static int ensure_scratch(Engine::Impl* d, size_t bytes)
{
    if (bytes <= d->scratch_bytes) return 0;
    if (d->d_scratch) cudaFree(d->d_scratch);
    d->scratch_bytes = 0;
    if (cudaMalloc(&d->d_scratch, bytes) != cudaSuccess) return -1;
    d->scratch_bytes = bytes;
    return 0;
}

int Engine::render_scans(const double* pts, const int64_t* offsets, int n_scans, const double* origins, const double* quats, const SE2* states, bool full,
                         uint64_t* cells)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (!d_->view.kbits || cfg_.occupancy_kind != 0) return fail("render_scans: needs a frequency map with a known plane", LAMA_ERR_STATE);
    if (n_scans < 0 || (n_scans && (!offsets || !states))) return fail("render_scans: bad arguments", LAMA_ERR_ARG);
    if (cells) *cells = 0;
    if (n_scans == 0) return LAMA_OK;
    if (offsets[0] != 0) return fail("render_scans: offsets[0] must be 0", LAMA_ERR_ARG);
    for (int k = 0; k < n_scans; ++k)
        if (offsets[k + 1] < offsets[k]) return fail("render_scans: offsets must not decrease", LAMA_ERR_ARG);
    const int64_t n_pts = offsets[n_scans];
    if (n_pts && !pts) return fail("render_scans: null points", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    std::vector<MovingTf> moving((size_t)n_scans);
    for (int k = 0; k < n_scans; ++k) moving[k] = moving_tf(origins ? origins + 3 * (size_t)k : nullptr, quats ? quats + 4 * (size_t)k : nullptr);
    // scratch: points | offsets | moving | states | marks (dim^2 bytes) | cell counter
    auto up = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    const size_t b_pts = up((size_t)n_pts * 24), b_off = up((size_t)(n_scans + 1) * 8), b_mov = up((size_t)n_scans * sizeof(MovingTf)),
                 b_st = up((size_t)n_scans * sizeof(SE2)), b_marks = up(dim2);
    if (ensure_scratch(d_, b_pts + b_off + b_mov + b_st + b_marks + 16)) return fail("render_scans: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch;
    RenderParams p;
    p.points  = (const double*)base;
    p.offsets = (const int64_t*)(base + b_pts);
    p.moving  = (const MovingTf*)(base + b_pts + b_off);
    p.states  = (const SE2*)(base + b_pts + b_off + b_mov);
    p.marks   = (uint8_t*)(base + b_pts + b_off + b_mov + b_st);
    p.cells   = (unsigned long long*)(base + b_pts + b_off + b_mov + b_st + b_marks);
    p.scale   = 1.0 / cfg_.resolution;
    p.full    = full ? 1 : 0;
    if (n_pts) CU_TRY(cudaMemcpyAsync((void*)p.points, pts, (size_t)n_pts * 24, cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaMemcpyAsync((void*)p.offsets, offsets, (size_t)(n_scans + 1) * 8, cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaMemcpyAsync((void*)p.moving, moving.data(), (size_t)n_scans * sizeof(MovingTf), cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaMemcpyAsync((void*)p.states, states, (size_t)n_scans * sizeof(SE2), cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaMemsetAsync(p.marks, 0, b_marks + 16, d_->stream));   // marks and the cell counter
    h2d_bytes_ += (uint64_t)n_pts * 24;
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    launch_render_scans(d_->view, cur_set_, p, n_scans, d_->stream);
    CU_TRY(cudaGetLastError());
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    unsigned long long n_cells = 0;
    CU_TRY(cudaMemcpyAsync(&n_cells, p.cells, 8, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_) {
        float ms = 0.f;
        CU_TRY(cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]));
        times_.raycast_ms += ms;
    }
    times_.raycast_launches += 4;
    if (cells) *cells = n_cells;
    return check_device_status();
}

int Engine::prune_frequency()
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (!d_->view.kbits || cfg_.occupancy_kind != 0) return fail("prune_frequency: needs a frequency map with a known plane", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    launch_prune_freq(d_->view, cur_set_, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return check_device_status();
}

int Engine::dm_apply(int particle, const uint32_t* cells_xy, const uint8_t* is_add, int n, uint32_t* processed)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || n < 0) return fail("dm_apply: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    uint32_t total = 0;
    const int cap = d_->ray.event_cap;
    std::vector<uint64_t> ev;
    int done = 0;
    do {  // One brushfire over the whole list reproduces the reference (all cells queued, then ONE update()).  Lists longer than the
          // per-particle event buffer (2 048 cells: the waves they start already fill most of the 8 192-entry heap in shared
          // memory) are applied in pieces with a brushfire after each, which gives a valid distance map but not necessarily the
          // reference's tie order -- big maps are loaded with lama_dm_read / lama_dm_import instead (DESIGN.md 10).
        int m = std::min(cap, n - done);
        ev.resize((size_t)std::max(m, 1));
        for (int i = 0; i < m; ++i) {
            uint32_t x = cells_xy[2 * (done + i)], y = cells_xy[2 * (done + i) + 1];
            if (dir_index(window_, x, y) < 0) return fail("dm_apply: cell outside the directory window", LAMA_ERR_WINDOW);
            ev[i] = push_record(((uint32_t)i << 1) | (is_add[done + i] ? 1u : 0u), cell_key(window_, x, y));
        }
        MapUpdateStats st{};
        st.events = (uint32_t)m;
        uint64_t* dev_ev = d_->d_events + (size_t)particle * cap;
        CU_TRY(cudaMemcpyAsync(dev_ev, ev.data(), (size_t)m * 8, cudaMemcpyHostToDevice, d_->stream));
        CU_TRY(cudaMemcpyAsync(d_->d_stats + particle, &st, sizeof(st), cudaMemcpyHostToDevice, d_->stream));
        BrushParams bp = d_->brush;
        bp.set = cur_set_;
        bp.particle_offset = particle;
        // block 0 of this launch must read the event list / stats of `particle`
        launch_brushfire(d_->view, bp, dev_ev, d_->d_stats + particle, 1, d_->stream);
        launch_merge_free(d_->view, d_->stream);
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(d_->h_stats, d_->d_stats + particle, sizeof(MapUpdateStats), cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));
        times_.brushfire_launches += 1;
        times_.misc_launches += 1;
        total += d_->h_stats[0].dm_pops;
        done += m;
        int rc = check_device_status();
        if (rc != LAMA_OK) return rc;
    } while (done < n);
    if (processed) *processed = total;
    return LAMA_OK;
}

int Engine::sampling_likelihood(int particle, const SE2& pose, const double* offsets_xy, int n, int stride, double* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || n < 1 || stride < 1) return fail("sampling_likelihood: bad arguments", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("sampling_likelihood: no scan uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    if (ensure_scratch(d_, (size_t)n * 24)) return fail("sampling_likelihood: out of device memory", LAMA_ERR_CUDA);
    double* d_off = (double*)d_->d_scratch;
    double* d_out = d_off + 2 * (size_t)n;
    CU_TRY(cudaMemcpyAsync(d_off, offsets_xy, (size_t)n * 16, cudaMemcpyHostToDevice, d_->stream));
    launch_sampling(d_->view, cur_set_, particle, d_->d_points, d_->scan, pose, d_off, n, stride, cfg_.resolution, max_sqdist_, d_out, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::dm_distance(int particle, const double* pts, int n, double* dist, double* grad)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || n < 1) return fail("dm_distance: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t bp = (size_t)n * 24, bd = (size_t)n * 8, bg = (size_t)n * 24;
    if (ensure_scratch(d_, bp + bd + bg)) return fail("dm_distance: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch;
    CU_TRY(cudaMemcpyAsync(base, pts, bp, cudaMemcpyHostToDevice, d_->stream));
    launch_distance(d_->view, cur_set_, particle, (const double*)base, n, cfg_.resolution, max_sqdist_, (double*)(base + bp),
                    grad ? (double*)(base + bp + bd) : nullptr, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(dist, base + bp, bd, cudaMemcpyDeviceToHost, d_->stream));
    if (grad) CU_TRY(cudaMemcpyAsync(grad, base + bp + bd, bg, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::export_window(int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, uint32_t* words, uint8_t* present)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || kind < 0 || kind > 1 || w < 1 || h < 1) return fail("export_window: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t bw = (size_t)w * h * 4, bpz = (size_t)w * h;
    if (ensure_scratch(d_, bw + bpz)) return fail("export_window: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch;
    launch_export(d_->view, cur_set_, particle, kind, x0, y0, w, h, (uint32_t*)base, (uint8_t*)(base + bw), d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(words, base, bw, cudaMemcpyDeviceToHost, d_->stream));
    if (present) CU_TRY(cudaMemcpyAsync(present, base + bw, bpz, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::gather_cells(int particle, int kind, const uint32_t* cells_xy, int n, uint32_t* words, uint8_t* flags)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || kind < 0 || kind > 1 || n < 0 || (n && (!cells_xy || !words || !flags)))
        return fail("gather_cells: bad arguments", LAMA_ERR_ARG);
    if (n == 0) return LAMA_OK;
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t bc = (size_t)n * 8, bw = (size_t)n * 4, bf = (size_t)n;
    if (ensure_scratch(d_, bc + bw + bf)) return fail("gather_cells: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch;
    CU_TRY(cudaMemcpyAsync(base, cells_xy, bc, cudaMemcpyHostToDevice, d_->stream));
    launch_gather_cells(d_->view, cur_set_, particle, kind, (const uint32_t*)base, n, (uint32_t*)(base + bc), (uint8_t*)(base + bc + bw), d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(words, base + bc, bw, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(flags, base + bc + bw, bf, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::export_bits(int particle, int plane, uint32_t x0, uint32_t y0, int w, int h, uint8_t* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || plane < 0 || plane > 1 || w < 1 || h < 1) return fail("export_bits: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    if (ensure_scratch(d_, (size_t)w * h)) return fail("export_bits: out of device memory", LAMA_ERR_CUDA);
    launch_export_bits(d_->view, plane, cur_set_, particle, x0, y0, w, h, (uint8_t*)d_->d_scratch, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, d_->d_scratch, (size_t)w * h, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::import_window(int particle, int kind, uint32_t x0, uint32_t y0, int w, int h, const uint32_t* words)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || kind < 0 || kind > 1 || w < 1 || h < 1 || (x0 | y0 | (uint32_t)w | (uint32_t)h) % kPatchLen)
        return fail("import_window: window must be patch aligned", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t bw = (size_t)w * h * 4;
    if (ensure_scratch(d_, bw)) return fail("import_window: out of device memory", LAMA_ERR_CUDA);
    CU_TRY(cudaMemcpyAsync(d_->d_scratch, words, bw, cudaMemcpyHostToDevice, d_->stream));
    launch_import(d_->view, cur_set_, particle, kind, x0, y0, w, h, (const uint32_t*)d_->d_scratch, d_->stream);
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 2;
    return check_device_status();
}

static const uint32_t kPackMagic = 0x4c414d50u;  // "LAMP"

int Engine::pack_size(int particle, size_t* bytes)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles) return fail("pack_size: bad particle", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    std::vector<int32_t> dir(2 * dim2);
    const int32_t* src = d_->view.dirs + (((size_t)cur_set_ * cfg_.particles + particle) * d_->view.n_kinds) * dim2;
    CU_TRY(cudaMemcpyAsync(dir.data(), src, 2 * dim2 * 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    size_t n = 0;
    for (int32_t v : dir) n += v >= 0;
    *bytes = 16 + ((n * 4 + 15) & ~(size_t)15) + n * (size_t)(kPatchBytes + 128);
    return LAMA_OK;
}

int Engine::migration_alloc(size_t bytes, void** dptr)
{
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t need = ((bytes ? bytes : 16) + 255) & ~(size_t)255;
    while (d_->mig_chunk < d_->mig_chunks.size() && d_->mig_off + need > d_->mig_chunks[d_->mig_chunk].second) {
        ++d_->mig_chunk;
        d_->mig_off = 0;
    }
    if (d_->mig_chunk == d_->mig_chunks.size()) {
        const size_t chunk = std::max(need, (size_t)64 << 20);
        void* p = nullptr;
        CU_TRY(cudaMalloc(&p, chunk));
        d_->mig_chunks.push_back({(char*)p, chunk});
        d_->mig_off = 0;
    }
    *dptr = d_->mig_chunks[d_->mig_chunk].first + d_->mig_off;
    d_->mig_off += need;
    return LAMA_OK;
}
void Engine::migration_reset()
{
    cudaSetDevice(cfg_.device);
    cudaStreamSynchronize(d_->stream);   // nothing enqueued on the engine's stream reads the arena any more
    d_->mig_chunk = 0;
    d_->mig_off   = 0;
}

// the directory indices at the head of a blob, padded so that the patches behind them stay 16-byte aligned (they are copied as uint4)
static size_t blob_entry_bytes(size_t n) { return (n * 4 + 15) & ~(size_t)15; }

// blob = n x u32 directory index (occupancy entries first, padded to 16 bytes) + n patches (4 KiB) + n x 128 B obstacle-mirror bits, all on the device
int Engine::pack_device(int particle, DeviceBlob* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles) return fail("pack: bad particle", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    std::vector<int32_t> dir(2 * dim2);
    const int32_t* src = d_->view.dirs + (((size_t)cur_set_ * cfg_.particles + particle) * d_->view.n_kinds) * dim2;
    CU_TRY(cudaMemcpyAsync(dir.data(), src, 2 * dim2 * 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    std::vector<int32_t> entries, slots;
    uint32_t n_kind[2] = {0, 0};
    for (int kind = 0; kind < 2; ++kind)
        for (size_t e = 0; e < dim2; ++e)
            if (dir[kind * dim2 + e] >= 0) {
                entries.push_back((int32_t)e);
                slots.push_back(dir[kind * dim2 + e]);
                ++n_kind[kind];
            }
    const size_t n = slots.size(), ne = blob_entry_bytes(n);
    out->n_occ = n_kind[0];
    out->n_dm  = n_kind[1];
    out->bytes = ne + n * (size_t)(kPatchBytes + 128);
    { int rc = migration_alloc(out->bytes + n * 4, &out->dptr); if (rc != LAMA_OK) return rc; }
    if (n) {
        char* base = (char*)out->dptr;
        uint32_t* d_out  = (uint32_t*)(base + ne);                                     // n patches, then n x 32 obstacle-mirror words
        uint32_t* d_fb   = (uint32_t*)(base + ne + n * (size_t)kPatchBytes);
        int32_t* d_slots = (int32_t*)(base + out->bytes);                              // scratch behind the blob
        CU_TRY(cudaMemcpyAsync(base, entries.data(), n * 4, cudaMemcpyHostToDevice, d_->stream));
        CU_TRY(cudaMemcpyAsync(d_slots, slots.data(), n * 4, cudaMemcpyHostToDevice, d_->stream));
        launch_gather_patches(d_->view, d_slots, (int)n, d_out, d_fb, nullptr, d_->stream);
        CU_TRY(cudaGetLastError());   // no synchronisation: `entries` / `slots` are pageable, the runtime has staged them when cudaMemcpyAsync returns
        times_.misc_launches += 1;
    }
    return LAMA_OK;
}

int Engine::unpack_device(int particle, const DeviceBlob& blob, bool check)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    const size_t n = (size_t)blob.n_occ + blob.n_dm, ne = blob_entry_bytes(n);
    if (particle < 0 || particle >= cfg_.particles || blob.bytes < ne + n * (size_t)(kPatchBytes + 128)) return fail("unpack: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    launch_release(d_->view, cur_set_, particle, 1, d_->stream);
    launch_merge_free(d_->view, d_->stream);
    if (n) {
        const char* base = (const char*)blob.dptr;
        const int32_t* d_entries = (const int32_t*)base;
        const uint32_t* d_in = (const uint32_t*)(base + ne);
        const uint32_t* d_fb = (const uint32_t*)(base + ne + n * (size_t)kPatchBytes);
        launch_scatter_patches(d_->view, cur_set_, particle, kMapOcc, d_entries, (int)blob.n_occ, d_in, d_fb, d_->stream);
        launch_scatter_patches(d_->view, cur_set_, particle, kMapDm, d_entries + blob.n_occ, (int)blob.n_dm, d_in + blob.n_occ * (size_t)kPatchCells,
                               d_fb + blob.n_occ * 32, d_->stream);
        times_.misc_launches += 2;
    }
    CU_TRY(cudaGetLastError());
    if (!check) return LAMA_OK;   // the caller unpacks several blobs and checks the device status after the last one
    CU_TRY(cudaMemcpyAsync(d_->h_status, d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    return check_device_status();
}

static uint32_t pack_window_word(int dir_dim, const DirWindow& w) { return (uint32_t)dir_dim | ((uint32_t)(w.base_px & 0xFFF) << 8) | ((uint32_t)(w.base_py & 0xFFF) << 20); }

// host form: {u32 magic, u32 dim + window base, u32 n_occ, u32 n_dm} + the device blob
int Engine::pack(int particle, void* buf, size_t cap, size_t* used)
{
    DeviceBlob blob;
    { int rc = pack_device(particle, &blob); if (rc != LAMA_OK) return rc; }
    const size_t need = 16 + blob.bytes;
    if (need > cap) { migration_reset(); return fail("pack: buffer too small", LAMA_ERR_ARG); }
    uint32_t* hdr = (uint32_t*)buf;
    // the directory indices in the buffer only mean the same cells on a device with the same window: dim and base travel along
    hdr[0] = kPackMagic; hdr[1] = pack_window_word(cfg_.dir_dim, window_); hdr[2] = blob.n_occ; hdr[3] = blob.n_dm;
    if (blob.bytes) {
        CU_TRY(cudaMemcpyAsync((char*)buf + 16, blob.dptr, blob.bytes, cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));
    }
    migration_reset();
    *used = need;
    return LAMA_OK;
}

int Engine::unpack(int particle, const void* buf, size_t bytes)
{
    if (particle < 0 || particle >= cfg_.particles || bytes < 16) return fail("unpack: bad arguments", LAMA_ERR_ARG);
    const uint32_t* hdr = (const uint32_t*)buf;
    if (hdr[0] != kPackMagic || hdr[1] != pack_window_word(cfg_.dir_dim, window_)) return fail("unpack: incompatible buffer (directory window differs)", LAMA_ERR_ARG);
    DeviceBlob blob;
    blob.n_occ = hdr[2];
    blob.n_dm  = hdr[3];
    const size_t n = (size_t)blob.n_occ + blob.n_dm;
    blob.bytes = blob_entry_bytes(n) + n * (size_t)(kPatchBytes + 128);
    if (bytes < 16 + blob.bytes) return fail("unpack: truncated buffer", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = migration_alloc(blob.bytes, &blob.dptr); if (rc != LAMA_OK) return rc; }
    if (blob.bytes) CU_TRY(cudaMemcpyAsync(blob.dptr, (const char*)buf + 16, blob.bytes, cudaMemcpyHostToDevice, d_->stream));
    const int rc = unpack_device(particle, blob);
    migration_reset();
    return rc;
}

double Engine::logodds_threshold() const { return d_->ray.prob.thresh; }
const ScanParams& Engine::scan_params() const { return d_->scan; }

int Engine::prune_outside(int particle, const double center[2], const double hwidth[2], int* removed)
{
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }
    if (particle < 0 || particle >= cfg_.particles) return fail("prune_outside: no such particle", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    std::vector<int32_t> dirs(2 * dim2);   // kinds 0 (occupancy) and 1 (distance) are adjacent
    const int32_t* src = d_->view.dirs + (((size_t)cur_set_ * cfg_.particles + particle) * d_->view.n_kinds) * dim2;
    CU_TRY(cudaMemcpyAsync(dirs.data(), src, 2 * dim2 * 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    const double scale = 1.0 / cfg_.resolution, off = (double)kMapOffsetCells;
    std::vector<int32_t> list;
    for (int py = 0; py < cfg_.dir_dim; ++py)
        for (int px = 0; px < cfg_.dir_dim; ++px) {
            const size_t di = (size_t)py * cfg_.dir_dim + px;
            // the reference walks the DISTANCE map's patches, which include every patch of the occupancy map (see capi.cpp: export_dm)
            if (dirs[di] < 0 && dirs[dim2 + di] < 0) continue;
            const uint32_t c0[2] = {(uint32_t)(window_.base_px + px) << kPatchLog2, (uint32_t)(window_.base_py + py) << kPatchLog2};
            bool meets = true;
            for (int k = 0; k < 2; ++k) {
                const double ws = ((double)c0[k] - off) / scale, we = ((double)(c0[k] + kPatchLen) - off) / scale;   // Map::m2w, map.h:147
                const double bh = (we - ws) * 0.5, bc = ws + bh;                                                        // AABB(min, max), aabb.h:50-55
                meets = meets && (std::abs(center[k] - bc) <= (hwidth[k] + bh));
            }
            if (!meets) list.push_back((int32_t)di);
        }
    if (removed) *removed = (int)list.size();
    if (list.empty()) return LAMA_OK;
    std::memcpy(d_->h_idx, list.data(), list.size() * 4);
    CU_TRY(cudaMemcpyAsync(d_->d_idx, d_->h_idx, list.size() * 4, cudaMemcpyHostToDevice, d_->stream));
    launch_delete_patches(d_->view, cur_set_, particle, d_->d_idx, (int)list.size(), d_->stream);
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 2;
    return LAMA_OK;
}

int Engine::bounds(int particle, int kind, uint32_t mn[2], uint32_t mx[2])
{
    if (settle(nullptr) != LAMA_OK) return -1;
    if (particle < 0 || particle >= cfg_.particles || kind < 0 || kind > 1) return -1;
    cudaSetDevice(cfg_.device);
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    std::vector<int32_t> dir(dim2);
    const int32_t* src = d_->view.dirs + (((size_t)cur_set_ * cfg_.particles + particle) * d_->view.n_kinds + kind) * dim2;
    if (cudaMemcpyAsync(dir.data(), src, dim2 * 4, cudaMemcpyDeviceToHost, d_->stream) != cudaSuccess) return -1;
    cudaStreamSynchronize(d_->stream);
    int n = 0;
    mn[0] = mn[1] = 0xffffffffu;
    mx[0] = mx[1] = 0;
    for (int py = 0; py < cfg_.dir_dim; ++py)
        for (int px = 0; px < cfg_.dir_dim; ++px)
            if (dir[(size_t)py * cfg_.dir_dim + px] >= 0) {
                uint32_t x = (uint32_t)(window_.base_px + px) << kPatchLog2, y = (uint32_t)(window_.base_py + py) << kPatchLog2;
                mn[0] = std::min(mn[0], x); mn[1] = std::min(mn[1], y);
                mx[0] = std::max(mx[0], x + kPatchLen); mx[1] = std::max(mx[1], y + kPatchLen);
                ++n;
            }
    return n;
}

int Engine::memory_usage(int kind, uint32_t cell_bytes, uint64_t* out)
{
    if (settle(nullptr) != LAMA_OK) return -1;
    if (kind < 0 || kind > 1 || !out) return -1;
    cudaSetDevice(cfg_.device);
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim, stride = (size_t)d_->view.n_kinds * dim2;
    std::vector<int32_t> dirs((size_t)cfg_.particles * stride), ref((size_t)d_->view.n_slots);
    const int32_t* src = d_->view.dirs + (size_t)cur_set_ * cfg_.particles * stride;
    if (cudaMemcpyAsync(dirs.data(), src, dirs.size() * 4, cudaMemcpyDeviceToHost, d_->stream) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(ref.data(), d_->view.refcount, ref.size() * 4, cudaMemcpyDeviceToHost, d_->stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(d_->stream) != cudaSuccess) return -1;
    const double container = (double)kPatchLen * kPatchLen * cell_bytes;
    for (int p = 0; p < cfg_.particles; ++p) {
        const int32_t* dir = dirs.data() + (size_t)p * stride + (size_t)kind * dim2;
        const int32_t* occ = dirs.data() + (size_t)p * stride;   // kind 0
        double total = 0.0;
        for (size_t e = 0; e < dim2; ++e) {
            // The reference's distance map also owns a patch wherever an occupancy cell was touched (the first touch of an occupancy cell reports
            // "changed" and calls removeObstacle, whose mutable get allocates -- and un-shares -- the distance patch: capi.cpp export_dm).  On the
            // device those cells live in the occupancy patch only, so a distance patch counts as shared by no more particles than the occupancy
            // patch over the same cells (which the ray cast un-shares on any touch, not only on first touches: an upper estimate of the bytes).
            int uses = 0;
            if (kind == 1) {
                const int ud = dir[e] >= 0 ? ref[(size_t)(dir[e] & kDirSlotMask)] : 0, uo = occ[e] >= 0 ? ref[(size_t)(occ[e] & kDirSlotMask)] : 0;
                if (ud <= 0 && uo <= 0) continue;
                uses = ud > 0 && uo > 0 ? std::min(ud, uo) : std::max(ud, uo);
            } else {
                if (dir[e] < 0) continue;
                uses = ref[(size_t)(dir[e] & kDirSlotMask)];
            }
            total += 72.0;
            total += container / (double)(uses > 0 ? uses : 1);
        }
        out[p] = (uint64_t)total;
    }
    return 0;
}

// ---- checkpoints --------------------------------------------------------------------------------------------------------------------
constexpr size_t kCkptChunk = (size_t)8 << 20;   // bytes per pinned buffer of the chunked copies (two of them)

namespace {
struct PinnedPair {   // two pinned chunk buffers and their completion events, released on every exit path
    char* buf[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    cudaError_t init()
    {
        for (int b = 0; b < 2; ++b) {
            cudaError_t e = cudaMallocHost((void**)&buf[b], kCkptChunk);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    ~PinnedPair()
    {
        for (int b = 0; b < 2; ++b) {
            if (done[b]) cudaEventSynchronize(done[b]), cudaEventDestroy(done[b]);
            if (buf[b]) cudaFreeHost(buf[b]);
        }
    }
};
struct DeviceAllocs {
    std::vector<void*> p;
    cudaError_t alloc(void** out, size_t bytes)
    {
        cudaError_t e = cudaMalloc(out, bytes ? bytes : 16);
        if (e == cudaSuccess) p.push_back(*out);
        return e;
    }
    ~DeviceAllocs() { for (void* q : p) cudaFree(q); }
};
double host_ms(std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); }
}  // namespace

int Engine::snapshot(EngineImage* out, CheckpointTimes* t)
{
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaSetDevice(cfg_.device));
    const StoreView& v = d_->view;
    const size_t n_slots = (size_t)v.n_slots, n_dir = (size_t)cfg_.particles * v.n_kinds * cfg_.dir_dim * cfg_.dir_dim;
    DeviceAllocs mem;
    CkptScratch c{};
    c.temp_bytes = ckpt_scan_temp_bytes(v.n_slots);
    CU_TRY(mem.alloc((void**)&c.cnt, n_slots * 4));
    CU_TRY(mem.alloc((void**)&c.used, n_slots * 4));
    CU_TRY(mem.alloc((void**)&c.new_id, n_slots * 4));
    CU_TRY(mem.alloc((void**)&c.list, n_slots * 4));
    CU_TRY(mem.alloc((void**)&c.ref, n_slots * 4));
    CU_TRY(mem.alloc((void**)&c.dirs, n_dir * 4));
    CU_TRY(mem.alloc((void**)&c.bad, 16));
    CU_TRY(mem.alloc(&c.temp, c.temp_bytes));
    cudaEvent_t ev[4] = {};
    struct Events { cudaEvent_t* e; ~Events() { for (int k = 0; k < 4; ++k) if (e[k]) cudaEventDestroy(e[k]); } } ev_guard{ev};
    for (int k = 0; k < 4; ++k) CU_TRY(cudaEventCreate(&ev[k]));
    CU_TRY(cudaMemsetAsync(c.cnt, 0, n_slots * 4, d_->stream));
    CU_TRY(cudaMemsetAsync(c.bad, 0, 4, d_->stream));
    CU_TRY(cudaEventRecord(ev[0], d_->stream));
    launch_ckpt_compact(v, cur_set_, c, d_->stream, ev[1]);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaEventRecord(ev[2], d_->stream));
    uint32_t bad = 0;
    int32_t last[2] = {0, 0};
    CU_TRY(cudaMemcpyAsync(&bad, c.bad, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(&last[0], c.new_id + n_slots - 1, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(&last[1], c.used + n_slots - 1, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 6;
    if (bad) return fail(bad & 1u ? "snapshot: a directory entry points outside the patch pool" : "snapshot: a patch's reference count differs from its directory references",
                         LAMA_ERR_STATE);
    const uint32_t K = (uint32_t)(last[0] + last[1]);

    EngineImage& img = *out;
    img.particles = cfg_.particles; img.dir_dim = cfg_.dir_dim; img.pool_slots = cfg_.pool_slots; img.max_beams = cfg_.max_beams;
    img.occupancy_kind = cfg_.occupancy_kind; img.known_plane = cfg_.known_plane; img.resolution = cfg_.resolution; img.l2_max = cfg_.l2_max;
    img.window = window_;
    img.used = K;
    const size_t stride = img.slot_stride(), bytes = (size_t)K * stride;
    char* stage = nullptr;
    CU_TRY(mem.alloc((void**)&stage, bytes));
    uint32_t* cells = (uint32_t*)stage;
    uint32_t* fb = (uint32_t*)(stage + (size_t)K * kPatchBytes);
    uint32_t* kb = img.has_kbits() ? (uint32_t*)(stage + (size_t)K * (kPatchBytes + 128)) : nullptr;
    launch_gather_patches(v, c.list, (int)K, cells, fb, kb, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaEventRecord(ev[3], d_->stream));
    if (K) times_.misc_launches += 1;
    img.refcount.resize(K);
    img.dirs.resize(n_dir);
    uint64_t cnt[3];
    CU_TRY(cudaMemcpyAsync(img.refcount.data(), c.ref, (size_t)K * 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(img.dirs.data(), c.dirs, n_dir * 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(cnt, v.counters, sizeof(cnt), cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    for (int k = 0; k < 3; ++k) img.counters[k] = cnt[k];

    // copy-out of the slots through two pinned chunk buffers: chunk i lands while the host copies chunk i - 1 away
    const auto t0 = std::chrono::steady_clock::now();
    img.slot_store.resize(bytes);
    img.slot_bytes = img.slot_store.data();
    PinnedPair pin;
    CU_TRY(pin.init());
    const size_t n_chunks = (bytes + kCkptChunk - 1) / kCkptChunk;
    for (size_t i = 0; i <= n_chunks; ++i) {
        if (i < n_chunks) {
            const size_t off = i * kCkptChunk, len = std::min(kCkptChunk, bytes - off);
            CU_TRY(cudaMemcpyAsync(pin.buf[i & 1], stage + off, len, cudaMemcpyDeviceToHost, d_->stream));
            CU_TRY(cudaEventRecord(pin.done[i & 1], d_->stream));
        }
        if (i > 0) {
            const size_t j = i - 1, off = j * kCkptChunk, len = std::min(kCkptChunk, bytes - off);
            CU_TRY(cudaEventSynchronize(pin.done[j & 1]));
            std::memcpy(img.slot_store.data() + off, pin.buf[j & 1], len);
        }
    }
    d2h_bytes_ += bytes + n_dir * 4 + (uint64_t)K * 4;
    if (t) {
        float a = 0, b = 0, g = 0;
        CU_TRY(cudaEventElapsedTime(&a, ev[0], ev[1]));
        CU_TRY(cudaEventElapsedTime(&b, ev[1], ev[2]));
        CU_TRY(cudaEventElapsedTime(&g, ev[2], ev[3]));
        t->count_ms = a; t->compact_ms = b; t->gather_ms = g;
        t->copy_ms = host_ms(t0);
    }
    return LAMA_OK;
}

Engine* Engine::restore(const EngineImage& img, int device, uint64_t stream, std::string& err, CheckpointTimes* t)
{
    const auto t0 = std::chrono::steady_clock::now();
    EngineConfig cfg;
    cfg.device = device; cfg.particles = img.particles; cfg.resolution = img.resolution; cfg.l2_max = img.l2_max; cfg.dir_dim = img.dir_dim;
    cfg.pool_slots = img.pool_slots; cfg.max_beams = img.max_beams; cfg.stream = stream; cfg.occupancy_kind = img.occupancy_kind;
    cfg.known_plane = img.known_plane;
    std::unique_ptr<Engine> e(create(cfg, err));
    if (!e) return nullptr;
    if (e->cfg_.pool_slots != img.pool_slots || img.used > (uint32_t)img.pool_slots) { err = "restore: pool size differs from the image"; return nullptr; }
    const double create_ms = host_ms(t0);
    // the saved window base, not one recomputed from a centre
    e->window_ = img.window;
    Impl* d = e->d_;
    StoreView& v = d->view;
    v.window = img.window;
    const uint32_t K = img.used;
    auto cu = [&](cudaError_t r, const char* what) {
        if (r != cudaSuccess) err = std::string("restore: ") + what + ": " + cudaGetErrorString(r);
        return r == cudaSuccess;
    };
    // k_init_store left every directory at -1, every count at 0 and the free stack as n_slots-1 .. 0 with slot 0 on top: the slots K ..
    // n_slots-1 are its lowest n_slots - K entries, the lowest slot on top
    const auto t1 = std::chrono::steady_clock::now();
    const int32_t free_count = v.n_slots - (int32_t)K;
    if (!cu(cudaMemcpyAsync(v.refcount, img.refcount.data(), (size_t)K * 4, cudaMemcpyHostToDevice, d->stream), "reference counts") ||
        !cu(cudaMemcpyAsync(v.dirs, img.dirs.data(), img.dirs.size() * 4, cudaMemcpyHostToDevice, d->stream), "directories") ||
        !cu(cudaMemcpyAsync(v.counters, img.counters, 3 * sizeof(uint64_t), cudaMemcpyHostToDevice, d->stream), "store counters") ||
        !cu(cudaMemcpyAsync(v.free_count, &free_count, 4, cudaMemcpyHostToDevice, d->stream), "free stack") ||
        !cu(cudaStreamSynchronize(d->stream), "synchronize"))
        return nullptr;
    const double tables_ms = host_ms(t1);
    // the slots straight into pool slots 0 .. K-1 and the planes behind them, through two pinned chunk buffers
    const auto t2 = std::chrono::steady_clock::now();
    const size_t bytes = (size_t)K * img.slot_stride();
    struct Region { char* dst; size_t len; } regions[3] = {{(char*)v.pool, (size_t)K * kPatchBytes}, {(char*)v.fbits, (size_t)K * 128},
                                                          {img.has_kbits() ? (char*)v.kbits : nullptr, img.has_kbits() ? (size_t)K * 128 : 0}};
    PinnedPair pin;
    if (!cu(pin.init(), "pinned buffers")) return nullptr;
    const size_t n_chunks = (bytes + kCkptChunk - 1) / kCkptChunk;
    for (size_t i = 0; i < n_chunks; ++i) {
        const size_t off = i * kCkptChunk, len = std::min(kCkptChunk, bytes - off);
        if (i >= 2 && !cu(cudaEventSynchronize(pin.done[i & 1]), "copy")) return nullptr;   // chunk i - 2 has left this buffer
        std::memcpy(pin.buf[i & 1], img.slot_bytes + off, len);
        size_t base = 0;
        for (const Region& r : regions) {   // the chunk may straddle the cells and the planes
            const size_t lo = std::max(off, base), hi = std::min(off + len, base + r.len);
            if (lo < hi && !cu(cudaMemcpyAsync(r.dst + (lo - base), pin.buf[i & 1] + (lo - off), hi - lo, cudaMemcpyHostToDevice, d->stream), "copy"))
                return nullptr;
            base += r.len;
        }
        if (!cu(cudaEventRecord(pin.done[i & 1], d->stream), "copy")) return nullptr;
    }
    if (!cu(cudaStreamSynchronize(d->stream), "synchronize")) return nullptr;
    e->h2d_bytes_ = 0;
    e->settled_counters_[0] = img.counters[0]; e->settled_counters_[1] = img.counters[1]; e->settled_counters_[2] = img.counters[2];
    e->settled_counters_[3] = (uint64_t)free_count;
    if (t) {
        *t = CheckpointTimes();
        t->create_ms = create_ms; t->tables_ms = tables_ms; t->copy_ms = host_ms(t2);
    }
    return e.release();
}

}  // namespace lama_b200
