// engine.cu -- device memory, stream and kernel pipeline behind the front ends.
#include "engine.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>

#include "cuda_owned.h"
#include "dm_follow.h"
#include "kernels.cuh"
#include "render_plan.h"

namespace lama_b200 {

#define CU_TRY(expr)                                                                                   \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(_e), LAMA_ERR_CUDA); \
    } while (0)

struct Engine::Impl {
    // streams first, events next, buffers last: members are destroyed buffers first, then events, then streams
    Stream stream;   // the caller's stream (EngineConfig::stream, borrowed) or one of the engine's own
    // particle groups of the grouped step (Engine::step_groups): group g owns the particles [g * P / G, (g + 1) * P / G) and a stream of
    // its own; an upload stream carries the scan and the predicted states.  Each group's kernels count patches into a counter block
    // of their own (d_gcnt[g]), so that a report holds that group's work of one scan exactly; settle() folds the blocks into
    // view.counters.  A map update on one stream is the one-group case, counting into view.counters itself.
    // h_grep[half][g] = {status, allocated, detached, freed, free slots, ...}; with G > 1 slot G = view.counters at the step.
    Stream gstream[kMaxGroups];
    Stream up_stream;
    Event ev_match, ev_sync;
    Event ev[2];
    Event ev_render[2];   // around one group of a following render (shift_window takes ev[0] / ev[1] between groups)
    // timing of a map update: per report buffer {before the match, after the match, after the ray stage, after the brushfire}; read when
    // that update is collected, so no host synchronisation is added.  evp_match: the update recorded a match (evp[half][0] is set).
    Event evp[2][4];
    Event ev_gmatch[kMaxGroups], ev_gdone[kMaxGroups];
    Event ev_up, ev_fork;
    // the store's arrays; view holds pointers into them (view.pool aligned out of pool_raw; grow_pool replaces the per-slot ones)
    DeviceArray<char> pool_raw;
    DeviceArray<uint32_t> fbits, kbits;
    DeviceArray<int32_t> refcount, free_slots, freed, free_count, dirs;   // free_count: 64 B, view.free_count .. view.counters
    DeviceArray<uint64_t> brush_spill;
    DeviceArray<RayPullHeader> pull_hdr;
    DeviceArray<PullEntry> pull_list;
    DeviceArray<uint32_t> pull_hits;
    DeviceArray<uint2> pull_tasks;
    DeviceArray<int32_t> pull_ctrl;
    StoreView view{};
    // scan
    double* d_points = nullptr;      // current scan (points into d_scan_buf or d_staged)
    DeviceArray<double> d_scan_buf;
    DeviceArray<double> d_staged;
    int staged_scans = 0, staged_beams = 0;
    ScanParams scan{};
    // per-launch staging
    DeviceArray<SE2> d_states;
    PinnedArray<SE2> h_states;
    DeviceArray<MatchResult> d_results;
    PinnedArray<MatchResult> h_results;
    DeviceArray<MapUpdateStats> d_stats;
    PinnedArray<MapUpdateStats> h_stats;   // two halves (ping-pong between consecutive map updates)
    PinnedArray<double> h_scan;            // staging of a host scan (step_async)
    DeviceArray<uint64_t> d_events;
    DeviceArray<int32_t> d_idx;
    PinnedArray<int32_t> h_idx;
    PinnedArray<uint32_t> h_status;
    RayParams ray{};
    BrushParams brush{};
    int n_sms = 132;
    int pull_max_particles = 0;   // the pull form of the ray cast is used up to this many particles per device; 0 = never (the walk is not slower at any
                                  // count, see launch_ray_stage); LAMA_PULL_MAX_PARTICLES overrides
    bool scan_flat = false;     // the current scan has z == 0 everywhere and a sensor that keeps z planes: every beam is planar
    bool staged_flat = false;   // the same for the staged scans
    bool evp_used[2] = {false, false}, evp_match[2] = {false, false};
    int groups = 1;
    DeviceArray<uint64_t> d_gcnt;               // [kMaxGroups][4]
    PinnedArray<uint64_t> h_grep;               // [2][kMaxGroups + 1][8]
    int report_groups[2] = {0, 0};              // groups of the map update that reported into each half
    bool fork = true;                           // the group streams must wait for the launching stream before their next work
    bool groups_ran = false;                    // grouped steps since the last fold: d_gcnt and the deferred k_merge_free are pending
    int scan_half = 0;                          // half of d_scan_buf the last grouped host scan went to
    uint64_t scan_alloc = 0, prev_alloc = 0;    // patches the last booked grouped scan allocated (allocated + detached), and the sum at its booking
    // scratch for import/export/distance
    DeviceArray<char> d_scratch;
    // scratch of shift_window, apart from d_scratch: a following render shifts the window between groups while its scans sit in d_scratch
    DeviceArray<char> d_shift_scratch;
    // the dense directory of match_extent (Engine::extent_)
    DeviceArray<char> d_extent;
    // fleet rounds (fleet_reserve): room for fleet_cap scans of max_beams beams; the pinned staging h_fleet holds the descriptors, then
    // the points, in the layout of d_fleet; the per-block scan indices (upload_states' growth) and the sampling offsets and likelihoods
    DeviceArray<char> d_fleet;
    PinnedArray<char> h_fleet;
    int fleet_cap = 0, fleet_max_beams = 0;
    DeviceArray<int32_t> d_fleet_blocks;
    PinnedArray<int32_t> h_fleet_blocks;
    DeviceArray<double> d_fleet_off;
    DeviceArray<double> d_fleet_lik;
    PinnedArray<double> h_fleet_lik;
    int fleet_n_off = 0;
    FleetScan* fleet_scans() const { return (FleetScan*)d_fleet.get(); }
    double* fleet_points() const { return (double*)(d_fleet.get() + (size_t)fleet_cap * sizeof(FleetScan)); }
    // device arena of a migration round (pack_device / migration_alloc): bump allocation out of chunks that are kept between rounds, so that a resampling
    // scan costs no cudaMalloc / cudaFree once the arena has grown to its working size
    std::vector<DeviceArray<char>> mig_chunks;
    size_t mig_chunk = 0, mig_off = 0;
    // parked entries (window_shift_core.h): per set one device arena (park[set]) and the {offset, length} of every list, on the device
    // (d_park_ol[set]) and here; they change only in shift_window, resample and prune_outside
    DeviceArray<ParkEntry> park[2];
    DeviceArray<int2> d_park_ol[2];
    std::vector<int2> park_ol[2];
    uint64_t shifts = 0, restored = 0;
    ParkView pv(int set) const { return ParkView{park[set].get(), d_park_ol[set].get()}; }
    int n_lists() const { return (int)park_ol[0].size(); }
    size_t parked(int set) const
    {
        size_t n = 0;
        for (const int2& o : park_ol[set]) n += (size_t)o.y;
        return n;
    }
    cudaError_t fetch(int set, size_t list, std::vector<ParkEntry>& out)   // one parked list, synchronously
    {
        const int2 ol = park_ol[set][list];
        out.resize((size_t)ol.y);
        if (!ol.y) return cudaSuccess;
        cudaError_t e = cudaMemcpyAsync(out.data(), park[set].get() + ol.x, out.size() * sizeof(ParkEntry), cudaMemcpyDeviceToHost, stream);
        return e == cudaSuccess ? cudaStreamSynchronize(stream) : e;
    }
    void drop_arena(int set)   // the stream must have passed every use of the arena
    {
        park[set].reset();
        std::fill(park_ol[set].begin(), park_ol[set].end(), make_int2(0, 0));
        cudaMemsetAsync(d_park_ol[set].get(), 0, park_ol[set].size() * sizeof(int2), stream);
    }
    int launch_ray_stage(const StoreView& v, RayParams rp, const SE2* states, uint64_t* events, MapUpdateStats* stats, int count, cudaStream_t st) const;
};


constexpr int kPullMaxBeams = 4096;   // k_ray_setup sorts the beams of a scan in shared memory
constexpr int kGroupMinParticles = 256;   // particle groups of step_async from this many particles per device on: measured at 256 only
constexpr int kDefaultGroups     = 4;     // scripts/pf_groups_rate.py, DESIGN.md 7a

static bool points_flat(const double* pts, size_t n)
{
    for (size_t i = 0; i < n; ++i)
        if (pts[3 * i + 2] != 0.0) return false;
    return true;
}

// The occupancy ray cast of `count` particles.  Scans whose beams all start in the same cell (no per-beam ray truncation) go through
// the pull form (k_ray_setup + k_ray_pull); k_raycast, the per-beam walk, takes everything else: LidarOdometry2D's and truncated rays,
// and -- decided per particle on the device -- scans of a tilted sensor (`flat` false: the beams may leave the z plane).
int Engine::Impl::launch_ray_stage(const StoreView& v, RayParams rp, const SE2* states, uint64_t* events, MapUpdateStats* stats, int count,
                                   cudaStream_t st) const   // returns the number of kernels launched
{
    const ScanParams& sp = rp.scan;
    // The walk runs one CTA per particle, the pull form spreads the patches of all particles over every SM.  Measured on an H100 (scripts/pull_variants.py,
    // revisit regime): walk 0.152 / 0.200 / 0.318 / 0.636 ms, pull 0.227 / 0.287 / 0.393 / 0.632 ms at 32 / 64 / 128 / 256 particles -- the walk wins
    // up to 128 and ties at 256, so pull_max_particles defaults to 0; LAMA_PULL_MAX_PARTICLES (read when the engine is created) selects the pull
    // form up to that many particles per device.
    const bool no_pull = count > pull_max_particles;
    const bool flat = scan_flat && sp.moving.l[6] == 0.0 && sp.moving.l[7] == 0.0;
    rp.pull_fallback = 0;
    if (!no_pull && !sp.lo_ray && sp.truncated_ray == 0.0 && sp.n_beams <= kPullMaxBeams) {
        launch_raycast_pull(v, rp, states, events, stats, count, n_sms, st);
        if (flat) return 2;   // hit.z == start.z exactly for every beam: k_ray_setup takes every particle
        rp.pull_fallback = 1;
    }
    launch_raycast(v, rp, states, events, stats, count, st);
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

bool Engine::reach_fits(double resolution, double l2_max, uint32_t* radius, std::string& err)
{
    const double r = std::ceil(l2_max * (1.0 / resolution));
    if (!(resolution > 0) || !(r >= 0 && r <= kDmMaxRadius)) {
        err = "l2_max / resolution exceeds 63 cells (packed distance cell limit)";
        return false;
    }
    *radius = (uint32_t)r;
    return true;
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
    uint32_t radius = 0;
    if (!reach_fits(cfg.resolution, cfg.l2_max, &radius, err)) return nullptr;
    std::unique_ptr<Engine> e(new Engine());
    e->cfg_ = cfg;
    e->max_sqdist_ = radius * radius;
    if (e->cfg_.pool_slots <= 0) e->cfg_.pool_slots = auto_pool_slots(cfg.particles);
    if (e->cfg_.pool_slots >= kDirSlotMask) {   // directory entries keep the slot in 24 bits, all ones = "not writable"
        err = "pool_slots must be below 2^24 - 1 (the slot field of a directory entry)";
        return nullptr;
    }
    Impl* d = e->d_ = new Impl();
    auto bail = [&](const std::string& m) {
        err = m;
        return (Engine*)nullptr;
    };
#define CU_NEW(expr)                                                             \
    do {                                                                         \
        cudaError_t _e = (expr);                                                 \
        if (_e != cudaSuccess) return bail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
    CU_NEW(cudaSetDevice(cfg.device));
    if (cfg.stream)
        d->stream.borrow(reinterpret_cast<cudaStream_t>(cfg.stream));
    else
        CU_NEW(d->stream.create());
    CU_NEW(d->ev[0].create(cudaEventDefault));
    CU_NEW(d->ev[1].create(cudaEventDefault));
    CU_NEW(d->ev_render[0].create(cudaEventDefault));
    CU_NEW(d->ev_render[1].create(cudaEventDefault));
    for (int b = 0; b < 2; ++b)
        for (int k = 0; k < 4; ++k) CU_NEW(d->evp[b][k].create(cudaEventDefault));

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
    // k_raycast ORs cell offsets into patch base addresses: the pool starts on a 4 KiB boundary (cudaMalloc only promises 256 B)
    CU_NEW(d->pool_raw.alloc(((size_t)v.n_slots + 1) * kPatchBytes));
    v.pool = reinterpret_cast<uint32_t*>(((uintptr_t)d->pool_raw.get() + (kPatchBytes - 1)) & ~(uintptr_t)(kPatchBytes - 1));
    CU_NEW(d->fbits.alloc((size_t)v.n_slots * 32));
    v.fbits = d->fbits.get();
    if (cfg.occupancy_kind == 1 || cfg.known_plane) CU_NEW(d->kbits.alloc((size_t)v.n_slots * 32));
    v.kbits = d->kbits.get();
    CU_NEW(d->refcount.alloc((size_t)v.n_slots));
    CU_NEW(d->free_slots.alloc((size_t)v.n_slots));
    CU_NEW(d->freed.alloc((size_t)v.n_slots));
    CU_NEW(d->free_count.alloc(16));
    v.refcount    = d->refcount.get();
    v.free_slots  = d->free_slots.get();
    v.freed       = d->freed.get();
    v.free_count  = d->free_count.get();
    v.freed_count = v.free_count + 1;
    v.status      = reinterpret_cast<uint32_t*>(v.free_count + 2);
    v.counters    = reinterpret_cast<uint64_t*>(v.free_count + 4);
    CU_NEW(d->dirs.alloc(2 * (size_t)cfg.particles * v.n_kinds * dim2));
    v.dirs = d->dirs.get();
    for (int set = 0; set < 2; ++set) {
        d->park_ol[set].assign((size_t)cfg.particles * v.n_kinds, make_int2(0, 0));
        CU_NEW(d->d_park_ol[set].alloc(d->park_ol[set].size()));
        CU_NEW(cudaMemset(d->d_park_ol[set].get(), 0, d->park_ol[set].size() * sizeof(int2)));
    }
    // two halves: a grouped step uploads the next host scan into one while the other groups' ray casts may still read the other
    CU_NEW(d->d_scan_buf.alloc(2 * (size_t)cfg.max_beams * 3));
    d->d_points = d->d_scan_buf.get();

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
    // The brushfire heaps start in shared memory (8 192 lower and 2 048 raise entries, sized with the L1 the kernel's prefetch
    // needs) and move, when a push finds one full, to a per-particle region in global memory of 65 536 entries each: the
    // capacities of the host emulation that the CPU tests run against the reference, seven times the largest lower heap
    // measured on the synthetic datasets (9 344 at 0.015 m with a 61-cell reach).  1 MiB per particle.
    d->brush.lower_cap   = 8192;
    d->brush.raise_cap   = 2048;
    d->brush.lower_total = 65536;
    d->brush.raise_total = 65536;
    if (const char* hc = std::getenv("LAMA_BRUSH_HEAP_CAP")) {   // test hook: total entries of each heap (overflow at a small size)
        const int v = std::max(2, std::min(65536, std::atoi(hc))) & ~1;
        d->brush.lower_total = d->brush.raise_total = v;
    }
    if (const char* sc = std::getenv("LAMA_BRUSH_SMEM_HEAP")) {  // test hook: shared entries of each heap (forces the spill to global memory)
        const int v = std::max(2, std::atoi(sc)) & ~1;
        d->brush.lower_cap = std::min(d->brush.lower_cap, v);
        d->brush.raise_cap = std::min(d->brush.raise_cap, v);
    }
    d->brush.lower_cap = std::min(d->brush.lower_cap, d->brush.lower_total);
    d->brush.raise_cap = std::min(d->brush.raise_cap, d->brush.raise_total);
    CU_NEW(d->brush_spill.alloc((size_t)cfg.particles * (d->brush.lower_total + 2 + d->brush.raise_total + 2)));
    d->brush.lower_spill = d->brush_spill.get();
    d->brush.raise_spill = d->brush.lower_spill + (size_t)cfg.particles * (d->brush.lower_total + 2);
    d->brush.max_sqdist = e->max_sqdist_;
    CU_NEW(d->d_events.alloc((size_t)cfg.particles * d->ray.event_cap));
    {   // scratch of the pull ray cast (k_ray_setup -> k_ray_pull)
        RayPullView& pv = d->ray.pull;
        pv.stride = (std::min(cfg.max_beams, kPullMaxBeams) + 31) & ~31;
        if (pv.stride < 32) pv.stride = 32;
        int npad = 32;
        while (npad < pv.stride) npad <<= 1;
        pv.stride = npad;   // k_ray_setup writes whole sorted arrays of next_pow2(beams) entries
        CU_NEW(d->pull_hdr.alloc((size_t)cfg.particles));
        CU_NEW(d->pull_list.alloc((size_t)cfg.particles * pv.stride));
        CU_NEW(d->pull_hits.alloc((size_t)cfg.particles * pv.stride));
        CU_NEW(d->pull_tasks.alloc((size_t)cfg.particles * dim2));
        CU_NEW(d->pull_ctrl.alloc(16));
        pv.hdr   = d->pull_hdr.get();
        pv.list  = d->pull_list.get();
        pv.hits  = d->pull_hits.get();
        pv.tasks = d->pull_tasks.get();
        pv.ctrl  = d->pull_ctrl.get();
        CU_NEW(cudaMemset(pv.ctrl, 0, 64));
        CU_NEW(cudaMemset(pv.hdr, 0, (size_t)cfg.particles * sizeof(RayPullHeader)));
        v.ray_ctrl = pv.ctrl;
        int sms = 0;
        CU_NEW(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg.device));
        d->n_sms = sms > 0 ? sms : 132;
        if (const char* pm = std::getenv("LAMA_PULL_MAX_PARTICLES")) d->pull_max_particles = std::atoi(pm);
    }
    CU_NEW(d->d_stats.alloc((size_t)cfg.particles));
    const size_t idx_ints = std::max((size_t)cfg.particles, (size_t)cfg.dir_dim * cfg.dir_dim);   // resample indices / directory entries to delete
    CU_NEW(d->d_idx.alloc(idx_ints));
    CU_NEW(d->h_stats.alloc(2 * (size_t)cfg.particles));
    CU_NEW(d->h_grep.alloc(2 * (size_t)(kMaxGroups + 1) * 8));
    std::memset(d->h_grep.get(), 0, 2 * (size_t)(kMaxGroups + 1) * 8 * sizeof(uint64_t));
    CU_NEW(d->h_scan.alloc((size_t)cfg.max_beams * 3));
    CU_NEW(d->ev_match.create(cudaEventDisableTiming));
    CU_NEW(d->ev_sync.create(cudaEventDisableTiming));
    CU_NEW(d->h_idx.alloc(idx_ints));
    CU_NEW(d->h_status.alloc(16));

    // Particle groups of step_async (DESIGN.md 7a): a scan of G groups overlaps one group's brushfire and next match with other groups'
    // ray casts.  One group when the pull ray cast may be selected (its task list is shared by every particle of a launch); otherwise
    // kDefaultGroups from kGroupMinParticles particles on, measured by scripts/pf_groups_rate.py.  Developer hook, read here:
    // LAMA_PF_GROUPS sets G.
    {
        int g = cfg.particles >= kGroupMinParticles ? kDefaultGroups : 1;
        if (const char* pg = std::getenv("LAMA_PF_GROUPS")) g = std::atoi(pg);
        if (d->pull_max_particles > 0) g = 1;
        d->groups = std::max(1, std::min(std::min(g, kMaxGroups), cfg.particles));
        if (d->groups > 1) {
            for (int k = 0; k < d->groups; ++k) {
                CU_NEW(d->gstream[k].create());
                CU_NEW(d->ev_gmatch[k].create(cudaEventDisableTiming));
                CU_NEW(d->ev_gdone[k].create(cudaEventDisableTiming));
            }
            CU_NEW(d->up_stream.create());
            CU_NEW(d->ev_up.create(cudaEventDisableTiming));
            CU_NEW(d->ev_fork.create(cudaEventDisableTiming));
            CU_NEW(d->d_gcnt.alloc((size_t)kMaxGroups * 4));
            CU_NEW(cudaMemset(d->d_gcnt.get(), 0, (size_t)kMaxGroups * 4 * sizeof(uint64_t)));
        }
    }

    const size_t need_ray = raycast_smem_bytes(cfg.dir_dim, d->ray), need_match = match_smem_bytes(cfg.dir_dim, e->max_sqdist_),
                 need_brush = brushfire_smem_bytes(cfg.dir_dim, d->brush);
    if (need_ray > 227 * 1024 || need_match > 227 * 1024 || need_brush > 227 * 1024) return bail("shared memory budget exceeded (reduce max_beams / dir_dim)");
    CU_NEW(configure_kernels(cfg.dir_dim, e->max_sqdist_, d->ray, d->brush));

    launch_init_store(v, 2, d->stream);
    CU_NEW(cudaGetLastError());
    CU_NEW(cudaStreamSynchronize(d->stream));
#undef CU_NEW
    return e.release();
}

Engine::~Engine()
{
    if (!d_) return;
    cudaSetDevice(cfg_.device);
    for (cudaStream_t s : {d_->stream.get(), d_->up_stream.get()})
        if (s) cudaStreamSynchronize(s);
    for (const Stream& s : d_->gstream)
        if (s) cudaStreamSynchronize(s);
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
    d_->d_points = d_->d_scan_buf.get();
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
    CU_TRY(d_->d_staged.alloc((size_t)n_scans * n * 3));
    CU_TRY(cudaMemcpyAsync(d_->d_staged.get(), pts, (size_t)n_scans * n * 24, cudaMemcpyHostToDevice, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    d_->staged_scans = n_scans;
    d_->staged_beams = n;
    d_->staged_flat  = points_flat(pts, (size_t)n_scans * n);
    return LAMA_OK;
}

int Engine::select_staged(int index, const double origin[3], const double quat[4], double truncated_ray, double truncated_range)
{
    if (!d_->d_staged.get() || index < 0 || index >= d_->staged_scans) return fail("select_staged: no such staged scan", LAMA_ERR_ARG);
    set_moving(origin, quat, truncated_ray, truncated_range, d_->staged_beams);
    d_->d_points = d_->d_staged.get() + (size_t)index * d_->staged_beams * 3;
    d_->scan_flat = d_->staged_flat;
    return LAMA_OK;
}

int Engine::ensure_states(int count)
{
    if ((size_t)count <= d_->h_results.size()) return LAMA_OK;   // allocated last: the other three hold as many
    d_->d_states.reset(); d_->d_results.reset(); d_->h_states.reset(); d_->h_results.reset();
    const size_t cap = (size_t)std::max(count, cfg_.particles);
    CU_TRY(d_->d_states.alloc(cap));
    CU_TRY(d_->d_results.alloc(cap));
    CU_TRY(d_->h_states.alloc(cap));
    CU_TRY(d_->h_results.alloc(cap));
    return LAMA_OK;
}

// The predicted states through the pinned staging buffer into d_states, on `stream`
int Engine::upload_states(const SE2* states, int count, void* stream)
{
    { int rc = ensure_states(count); if (rc != LAMA_OK) return rc; }
    std::memcpy(d_->h_states.get(), states, (size_t)count * sizeof(SE2));
    CU_TRY(cudaMemcpyAsync(d_->d_states.get(), d_->h_states.get(), (size_t)count * sizeof(SE2), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    h2d_bytes_ += (uint64_t)count * sizeof(SE2);
    return LAMA_OK;
}

// A host scan through the pinned staging buffer into `dst`, on `stream`; it becomes the current scan.  The staging buffer is free: the
// previous step returned after its match, which follows its upload.
int Engine::upload_scan(const double* pts, int n, double* dst, void* stream)
{
    std::memcpy(d_->h_scan.get(), pts, (size_t)n * 24);
    d_->d_points = dst;
    d_->scan_flat = points_flat(pts, (size_t)n);
    CU_TRY(cudaMemcpyAsync(dst, d_->h_scan.get(), (size_t)n * 24, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    h2d_bytes_ += (uint64_t)n * 24;
    return LAMA_OK;
}

MatchParams Engine::match_params(const SolverOptions& so, double meas_sigma, int first_particle, bool shared_map, int mode) const
{
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
    mp.parked_any = d_->parked(cur_set_) != 0;
    return mp;
}

// developer builds (LAMA_PHASE_TIMING): LAMA_BF_DEBUG = ordinal of the map update whose k_brushfire prints its per-particle phase cycles
static int brush_debug_flag()
{
    static int launch_no = 0;
    const char* dbg = std::getenv("LAMA_BF_DEBUG");
    return dbg && std::atoi(dbg) == launch_no++;
}

// The brushfire of a map update with block 0 on `particle_offset` and, with `rp`, the ray cast of the current scan before it, reading
// poses `state_stride` bytes apart.  The ray cast's shared-memory scratch and the event lists are sized for this scan (two CTAs per SM
// at 1080 beams; the maxima were registered at create); a brushfire alone (dm_apply) takes lists of the full capacity.
BrushParams Engine::map_update_params(int state_stride, int particle_offset, RayParams* rp) const
{
    BrushParams bp = d_->brush;
    bp.set = cur_set_;
    bp.particle_offset = particle_offset;
    bp.debug = brush_debug_flag();
    if (!rp) return bp;
    *rp = d_->ray;
    rp->points = d_->d_points;
    rp->scan = d_->scan;
    rp->set = cur_set_;
    rp->particle_offset = particle_offset;
    rp->state_stride = state_stride;
    { const char* dbg = std::getenv("LAMA_RAY_DEBUG"); rp->debug = dbg ? std::atoi(dbg) : 0; }  // see RayParams::debug
    const int nb = d_->scan.n_beams;
    rp->log_cap   = std::min(d_->ray.log_cap, next_pow2_host(std::max(1024, 3 * nb)));
    rp->event_cap = std::min(d_->ray.event_cap, next_pow2_host(std::max(512, nb)));
    bp.event_cap = rp->event_cap;
    return bp;
}

int Engine::check_device_status()
{
    uint32_t st = *d_->h_status.get();
    if (!st) return LAMA_OK;
    if (st & kErrWindow) return fail("map grew outside the directory window (raise dir_dim)", LAMA_ERR_WINDOW);
    if (st & kErrPoolEmpty) return fail("patch pool exhausted (raise pool_slots)", LAMA_ERR_POOL);
    if (st & kErrHeapOverflow)
        return fail("brushfire heap overflow: a distance-map update queued more than " + std::to_string(d_->brush.lower_total) + " (lower) or " +
                        std::to_string(d_->brush.raise_total) + " (raise) cells at once",
                    LAMA_ERR_OVERFLOW);
    if (st & kErrPushOverflow)
        return fail("obstacle event list overflow: more addObstacle / removeObstacle calls in one map update than the per-particle list holds (" +
                        std::to_string(d_->brush.event_cap) + ")",
                    LAMA_ERR_OVERFLOW);
    return fail("ray-cast log overflow in the map update kernels", LAMA_ERR_OVERFLOW);
}

uint32_t Engine::device_status()
{
    settle(nullptr);
    cudaSetDevice(cfg_.device);
    cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream);
    cudaStreamSynchronize(d_->stream);
    return *d_->h_status.get();
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
    return match_sync(states, count, match_params(so, meas_sigma, first_particle, shared_map, mode), false, out);
}

// The synchronous match of match() and, with `extent`, of match_extent() (k_match_extent over its directory).  With parked entries a read
// outside the window sets kErrWindow (k_match reads it as absent): the caller must not get that result.
int Engine::match_sync(const SE2* states, int count, const MatchParams& mp, bool extent, HostMatchResult* out)
{
    { int rc = upload_states(states, count, d_->stream); if (rc != LAMA_OK) return rc; }
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    if (extent) launch_match_extent(d_->view, mp, (const int32_t*)d_->d_extent.get(), extent_, d_->d_states.get(), d_->d_results.get(), count, d_->stream);
    else launch_match(d_->view, mp, d_->d_states.get(), d_->d_results.get(), count, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_results.get(), d_->d_results.get(), (size_t)count * sizeof(MatchResult), cudaMemcpyDeviceToHost, d_->stream));
    if (mp.parked_any) CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_) {
        float ms = 0;
        cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]);
        times_.match_ms += ms;
    }
    times_.match_launches += 1;
    if (mp.parked_any && *d_->h_status.get()) return check_device_status();
    static_assert(sizeof(HostMatchResult) == sizeof(MatchResult), "layout");
    std::memcpy(out, d_->h_results.get(), (size_t)count * sizeof(MatchResult));
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
    { int rc = upload_states(states, count, d_->stream); if (rc != LAMA_OK) return rc; }
    double* d_out = reinterpret_cast<double*>(d_->d_results.get());   // count doubles fit in count MatchResults
    launch_match_error(d_->view, d_->pv(cur_set_), cur_set_, first_particle, shared_map, d_->d_points, d_->scan, d_->d_states.get(), count, cfg_.resolution, max_sqdist_, d_out, d_->stream);
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

// Launches ray cast + brushfire and returns without waiting; settle() (called by every later entry point)
// synchronises, collects the per-particle statistics and surfaces device errors.
int Engine::update_maps_async(const SE2* states, int first_particle, int count)
{
    extent_stale_ = true;
    if (count < 1 || first_particle < 0 || first_particle + count > cfg_.particles) return fail("update_maps: particle range out of bounds", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("update_maps: no scan uploaded", LAMA_ERR_STATE);
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = upload_states(states, count, d_->stream); if (rc != LAMA_OK) return rc; }
    RayParams rp;
    const BrushParams bp = map_update_params((int)sizeof(SE2), first_particle, &rp);
    { int rc = enqueue_group(nullptr, rp, bp, 0, count, d_->stream, d_->view.counters, 0, nullptr); if (rc != LAMA_OK) return rc; }
    const int half = 1 - pending_buf_;
    d_->report_groups[half] = 1;
    pending_buf_  = half;
    pending_maps_ = count;
    return LAMA_OK;
}

// Particles [lo, lo + cnt) of a map update on `stream`, their kernels counting patches into `counters` (view.counters on one stream, a
// group's block of d_gcnt in a grouped step): with `mp`, the match of their predicted states, the copy of its results to the host and
// `ev_match`, then the map update on the matched poses; without, the map update on the poses in d_states.  Then the ray stage, the
// brushfire, on one stream k_merge_free, and report g (statistics, status, counter block, free slots) into the half of the host buffers
// that the pending update does not use.  Timing mode (always one stream) records evp[half] around the kernels.
int Engine::enqueue_group(const MatchParams* mp, RayParams rp, BrushParams bp, int lo, int cnt, void* stream, uint64_t* counters, int g, void* ev_match)
{
    Impl* d = d_;
    cudaStream_t st = (cudaStream_t)stream;
    const int half = 1 - pending_buf_;
    const Event* ev = timing_ ? d->evp[half] : nullptr;
    StoreView v = d->view;
    v.counters = counters;
    const SE2* poses = d->d_states.get() + lo;
    if (mp) {
        MatchParams m = *mp;
        m.particle_offset += lo;
        if (ev) CU_TRY(cudaEventRecord(ev[0], st));
        launch_match(v, m, d->d_states.get() + lo, d->d_results.get() + lo, cnt, st);
        if (ev) CU_TRY(cudaEventRecord(ev[1], st));
        CU_TRY(cudaMemcpyAsync(d->h_results.get() + lo, d->d_results.get() + lo, (size_t)cnt * sizeof(MatchResult), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaEventRecord((cudaEvent_t)ev_match, st));
        poses = reinterpret_cast<const SE2*>(d->d_results.get() + lo);
        times_.match_launches += 1;
        d2h_bytes_ += (uint64_t)cnt * sizeof(MatchResult);
    } else if (ev) {
        CU_TRY(cudaEventRecord(ev[1], st));
    }
    uint64_t* events = d->d_events.get() + (size_t)lo * d->ray.event_cap;
    rp.particle_offset += lo;
    const int ray_kernels = d->launch_ray_stage(v, rp, poses, events, d->d_stats.get() + lo, cnt, st);
    if (ev) CU_TRY(cudaEventRecord(ev[2], st));
    bp.particle_offset += lo;
    bp.lower_spill += (size_t)lo * (d->brush.lower_total + 2);
    bp.raise_spill += (size_t)lo * (d->brush.raise_total + 2);
    launch_brushfire(v, bp, events, d->d_stats.get() + lo, cnt, st);
    if (ev) {
        CU_TRY(cudaEventRecord(ev[3], st));
        d->evp_used[half]  = true;
        d->evp_match[half] = mp != nullptr;
    }
    // a grouped step returns freed patches at the next barrier: k_merge_free is not safe beside another group's alloc_slot
    const bool one_stream = counters == d->view.counters;
    if (one_stream) launch_merge_free(d->view, st);
    CU_TRY(cudaGetLastError());
    uint64_t* r = d->h_grep.get() + ((size_t)half * (kMaxGroups + 1) + g) * 8;
    CU_TRY(cudaMemcpyAsync(d->h_stats.get() + (size_t)half * cfg_.particles + lo, d->d_stats.get() + lo, (size_t)cnt * sizeof(MapUpdateStats), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(r, d->view.status, 4, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(r + 1, counters, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(r + 4, d->view.free_count, 4, cudaMemcpyDeviceToHost, st));
    times_.raycast_launches += ray_kernels;
    times_.brushfire_launches += 1;
    times_.misc_launches += one_stream ? 1 : 0;
    d2h_bytes_ += (uint64_t)cnt * sizeof(MapUpdateStats) + 4 + 28;
    return LAMA_OK;
}

int Engine::check_step(const double* pts, int n, int count)
{
    if (count < 1 || count > cfg_.particles) return fail("step: particle range out of bounds", LAMA_ERR_ARG);
    if (pts && (n < 1 || n > cfg_.max_beams)) return fail("step: number of beams out of range", LAMA_ERR_ARG);
    if (!pts && d_->scan.n_beams < 1) return fail("step: no scan selected", LAMA_ERR_STATE);
    return LAMA_OK;
}

int Engine::step_enqueue(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                         const SE2* predicted, int count, const SolverOptions& so, double meas_sigma)
{
    { int rc = check_step(pts, n, count); if (rc != LAMA_OK) return rc; }
    extent_stale_ = true;
    d_->fork = true;   // a grouped step after this one waits for it
    CU_TRY(cudaSetDevice(cfg_.device));
    // the previous scan's map update may still be running: nothing below waits for it on the host
    enq_had_pending_ = pending_maps_ != 0;
    enq_prev_count_  = pending_maps_;
    enq_prev_buf_    = pending_buf_;
    if (pts) {
        set_moving(origin, quat, truncated_ray, truncated_range, n);
        int rc = upload_scan(pts, n, d_->d_scan_buf.get(), d_->stream);
        if (rc != LAMA_OK) return rc;
    }
    { int rc = upload_states(predicted, count, d_->stream); if (rc != LAMA_OK) return rc; }
    const MatchParams mp = match_params(so, meas_sigma, 0, false, 0);
    RayParams rp;
    const BrushParams bp = map_update_params((int)sizeof(MatchResult), 0, &rp);
    { int rc = enqueue_group(&mp, rp, bp, 0, count, d_->stream, d_->view.counters, 0, d_->ev_match); if (rc != LAMA_OK) return rc; }
    const int half = 1 - pending_buf_;
    d_->report_groups[half] = 1;
    pending_buf_  = half;
    pending_maps_ = count;
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

int Engine::particle_groups() const { return d_->groups; }

int Engine::step_async(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                       const SE2* predicted, int count, const SolverOptions& so, double meas_sigma, HostMatchResult* out)
{
    { int rc = check_step(pts, n, count); if (rc != LAMA_OK) return rc; }
    // timing mode keeps one stream, so that kernelTimes() still times single kernels
    if (d_->groups > 1 && count > 1 && !timing_) return step_groups(pts, n, origin, quat, truncated_ray, truncated_range, predicted, count, so, meas_sigma, out);
    { int rc = step_enqueue(pts, n, origin, quat, truncated_ray, truncated_range, predicted, count, so, meas_sigma); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaEventSynchronize(d_->ev_match));
    static_assert(sizeof(HostMatchResult) == sizeof(MatchResult), "layout");
    std::memcpy(out, d_->h_results.get(), (size_t)count * sizeof(MatchResult));
    return collect_previous();
}

// step_async over G particle groups (DESIGN.md 7a).  Group g's stream runs match -> copy of its results -> ray cast -> brushfire -> report of
// its particles; its particles' chain match(t) -> ray(t) -> brushfire(t) -> match(t + 1) depends on no other group, because the map update
// runs before the resampling decision, so the groups drift apart and one group's brushfire and next match run beside another group's
// ray cast.  The launching stream waits for every group at the end (its events keep meaning "this scan's
// map update has completed"); the groups wait for the launching stream only after settle(), which every other entry point calls first:
// that is the barrier behind which resampling, window shifts, checkpoints, exports and k_merge_free run.  Patches freed by a grouped
// scan go back to the free stack at the next barrier (k_merge_free is not safe beside a running alloc_slot), and a barrier is forced
// when the free stack drops under twice what the last booked scan allocated (at least one patch per particle and kind), so that
// freed patches waiting for the merge never make a scan run out of patches that one stream would have had.
int Engine::step_groups(const double* pts, int n, const double origin[3], const double quat[4], double truncated_ray, double truncated_range,
                        const SE2* predicted, int count, const SolverOptions& so, double meas_sigma, HostMatchResult* out)
{
    Impl* d = d_;
    if (d->groups_ran) {
        const uint64_t reserve = 2 * std::max<uint64_t>(d->scan_alloc, (uint64_t)count * d->view.n_kinds);
        if (settled_counters_[3] < reserve) {
            int rc = settle(nullptr);   // a barrier: the frees are merged, the groups fork again
            if (rc != LAMA_OK) return rc;
        }
    }
    extent_stale_ = true;
    CU_TRY(cudaSetDevice(cfg_.device));
    enq_had_pending_ = pending_maps_ != 0;
    enq_prev_count_  = pending_maps_;
    enq_prev_buf_    = pending_buf_;
    const int G = std::min(d->groups, count);
    if (d->fork) {   // work the engine put on the launching stream since the last grouped step comes first
        CU_TRY(cudaEventRecord(d->ev_fork, d->stream));
        CU_TRY(cudaStreamWaitEvent(d->up_stream, d->ev_fork, 0));
        for (int g = 0; g < d->groups; ++g) CU_TRY(cudaStreamWaitEvent(d->gstream[g], d->ev_fork, 0));
        d->fork = false;
    }
    // uploads: the scan goes to the half of d_scan_buf the previous scan did not use, since that scan's later ray casts may still be reading it
    if (pts) {
        set_moving(origin, quat, truncated_ray, truncated_range, n);
        d->scan_half ^= 1;
        int rc = upload_scan(pts, n, d->d_scan_buf.get() + (size_t)d->scan_half * cfg_.max_beams * 3, d->up_stream);
        if (rc != LAMA_OK) return rc;
    }
    { int rc = upload_states(predicted, count, d->up_stream); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaEventRecord(d->ev_up, d->up_stream));
    const MatchParams mp = match_params(so, meas_sigma, 0, false, 0);
    RayParams rp;
    const BrushParams bp = map_update_params((int)sizeof(MatchResult), 0, &rp);
    const int half = 1 - pending_buf_;
    for (int g = 0; g < G; ++g) {
        const int lo = (int)((int64_t)g * count / G), cnt = (int)((int64_t)(g + 1) * count / G) - lo;
        cudaStream_t st = d->gstream[g];
        CU_TRY(cudaStreamWaitEvent(st, d->ev_up, 0));
        { int rc = enqueue_group(&mp, rp, bp, lo, cnt, st, d->d_gcnt.get() + (size_t)g * 4, g, d->ev_gmatch[g]); if (rc != LAMA_OK) return rc; }
        if (g == 0) {   // view.counters, which no kernel of a grouped step writes, into slot G of the report
            CU_TRY(cudaMemcpyAsync(d->h_grep.get() + ((size_t)half * (kMaxGroups + 1) + G) * 8 + 1, d->view.counters, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
            d2h_bytes_ += 24;
        }
        CU_TRY(cudaEventRecord(d->ev_gdone[g], st));
    }
    for (int g = 0; g < G; ++g) CU_TRY(cudaStreamWaitEvent(d->stream, d->ev_gdone[g], 0));   // the launching stream joins every group
    d->groups_ran = true;
    d->report_groups[half] = G;
    pending_buf_  = half;
    pending_maps_ = count;
    for (int g = 0; g < G; ++g) CU_TRY(cudaEventSynchronize(d->ev_gmatch[g]));
    static_assert(sizeof(HostMatchResult) == sizeof(MatchResult), "layout");
    std::memcpy(out, d->h_results.get(), (size_t)count * sizeof(MatchResult));
    return collect_previous();
}

// Folds the groups' counter blocks into view.counters and returns the patches freed by grouped scans to the free stack.  The engine's
// streams must have completed (settle() calls it after synchronising the launching stream, which has joined every group).
int Engine::fold_groups()
{
    Impl* d = d_;
    d->groups_ran = false;
    uint64_t g[kMaxGroups * 4], m[3];
    CU_TRY(cudaMemcpyAsync(g, d->d_gcnt.get(), sizeof(g), cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(cudaMemcpyAsync(m, d->view.counters, sizeof(m), cudaMemcpyDeviceToHost, d->stream));
    CU_TRY(cudaStreamSynchronize(d->stream));
    for (int k = 0; k < kMaxGroups; ++k)
        for (int c = 0; c < 3; ++c) m[c] += g[k * 4 + c];
    CU_TRY(cudaMemcpyAsync(d->view.counters, m, sizeof(m), cudaMemcpyHostToDevice, d->stream));
    CU_TRY(cudaMemsetAsync(d->d_gcnt.get(), 0, sizeof(g), d->stream));
    launch_merge_free(d->view, d->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d->stream));   // `m` is on this stack
    times_.misc_launches += 1;
    return LAMA_OK;
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
    launch_pack_results(d_->d_results.get(), count, digest, d_out, st);
    CU_TRY(cudaGetLastError());
    return LAMA_OK;
}

int Engine::settle(HostMapStats* out, bool already_complete)
{
    if (!already_complete) d_->fork = true;   // whatever the caller enqueues next on the launching stream precedes the next grouped step
    if (pending_maps_ == 0) {
        if (!already_complete && d_->groups_ran) {
            CU_TRY(cudaSetDevice(cfg_.device));
            return fold_groups();
        }
        return LAMA_OK;
    }
    const int count = pending_maps_, half = pending_buf_;
    pending_maps_ = 0;
    CU_TRY(cudaSetDevice(cfg_.device));
    if (!already_complete) CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_ && d_->evp_used[half]) {   // the update's events have completed (the stream is past them, or was just synchronised)
        const Event* e = d_->evp[half];
        float m = 0, a = 0, b = 0;
        if (d_->evp_match[half]) cudaEventElapsedTime(&m, e[0], e[1]);
        cudaEventElapsedTime(&a, e[1], e[2]);
        cudaEventElapsedTime(&b, e[2], e[3]);
        times_.match_ms += m;
        times_.raycast_ms += a;
        times_.brushfire_ms += b;
        d_->evp_used[half] = false;
    }
    static_assert(sizeof(HostMapStats) == sizeof(MapUpdateStats), "layout");
    const MapUpdateStats* hs = d_->h_stats.get() + (size_t)half * cfg_.particles;
    last_map_stats_.assign((const HostMapStats*)hs, (const HostMapStats*)hs + count);
    if (out) std::memcpy(out, hs, (size_t)count * sizeof(MapUpdateStats));
    // view.counters plus every group's block; one group is a map update on one stream, whose block is view.counters itself
    const int G = d_->report_groups[half];
    const uint64_t* hr = d_->h_grep.get() + (size_t)half * (kMaxGroups + 1) * 8;
    uint32_t status = 0;
    for (int c = 0; c < 3; ++c) settled_counters_[c] = G > 1 ? hr[(size_t)G * 8 + 1 + c] : 0;
    for (int g = 0; g < G; ++g) {
        status |= (uint32_t)hr[g * 8];
        for (int c = 0; c < 3; ++c) settled_counters_[c] += hr[g * 8 + 1 + c];
    }
    settled_counters_[3] = (uint64_t)(uint32_t)hr[(G - 1) * 8 + 4];
    *d_->h_status.get() = status;
    if (G > 1) {
        const uint64_t alloc = settled_counters_[0] + settled_counters_[1];
        d_->scan_alloc = d_->prev_alloc && alloc > d_->prev_alloc ? alloc - d_->prev_alloc : 0;
        d_->prev_alloc = alloc;
    }
    if (!already_complete && d_->groups_ran) {
        int rc = fold_groups();
        if (rc != LAMA_OK) return rc;
    }
    return check_device_status();
}

int Engine::share_from(int src_particle, int dst_first, int count)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    extent_stale_ = true;
    if (count == 0) return LAMA_OK;
    if (src_particle < 0 || src_particle >= cfg_.particles || dst_first < 0 || dst_first + count > cfg_.particles ||
        (src_particle >= dst_first && src_particle < dst_first + count))
        return fail("share_from: bad particle range", LAMA_ERR_ARG);
    if (has_parked()) return fail("share_from: the maps have parked entries (the window has moved); share_from builds a filter's first maps", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    for (int i = 0; i < count; ++i) d_->h_idx.get()[i] = src_particle;
    CU_TRY(cudaMemcpyAsync(d_->d_idx.get(), d_->h_idx.get(), (size_t)count * 4, cudaMemcpyHostToDevice, d_->stream));
    launch_release(d_->view, cur_set_, dst_first, count, d_->stream);
    launch_copy_dirs(d_->view, cur_set_, cur_set_, d_->d_idx.get(), dst_first, count, d_->stream);
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 3;
    return LAMA_OK;
}

int Engine::resample(const int32_t* idx)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    extent_stale_ = true;
    CU_TRY(cudaSetDevice(cfg_.device));
    const int P = cfg_.particles;
    for (int i = 0; i < P; ++i) {
        if (idx[i] < -1 || idx[i] >= P) return fail("resample: index out of range", LAMA_ERR_ARG);
        d_->h_idx.get()[i] = idx[i];
    }
    CU_TRY(cudaMemcpyAsync(d_->d_idx.get(), d_->h_idx.get(), (size_t)P * 4, cudaMemcpyHostToDevice, d_->stream));
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    const int other = 1 - cur_set_;
    // the offspring's parked lists: copies of their ancestors' (kinds 0 and 1, like the directories), in a new arena of the other set
    const bool parked = d_->parked(cur_set_) != 0;
    if (parked) {
        const int nk = d_->view.n_kinds;
        std::vector<int2>& ol = d_->park_ol[other];
        int32_t off = 0;
        for (int p = 0; p < P; ++p)
            for (int k = 0; k < nk; ++k) {
                const int32_t len = idx[p] >= 0 && k < 2 ? d_->park_ol[cur_set_][(size_t)idx[p] * nk + k].y : 0;
                ol[(size_t)p * nk + k] = make_int2(off, len);
                off += len;
            }
        if (off) CU_TRY(d_->park[other].alloc((size_t)off));
        CU_TRY(cudaMemcpyAsync(d_->d_park_ol[other].get(), ol.data(), ol.size() * sizeof(int2), cudaMemcpyHostToDevice, d_->stream));
    }
    launch_copy_dirs(d_->view, cur_set_, other, d_->d_idx.get(), 0, P, d_->stream);  // share first ...
    if (parked && d_->park[other])
        launch_copy_parked(d_->view, d_->park[cur_set_].get(), d_->d_park_ol[cur_set_].get(), d_->park[other].get(), d_->d_park_ol[other].get(), d_->d_idx.get(), P,
                           d_->stream);
    launch_release(d_->view, cur_set_, 0, P, d_->stream);                       // ... then drop the old set
    launch_release_parked(d_->view, d_->pv(cur_set_), 0, P, d_->stream);
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
    if (parked) {
        d_->drop_arena(cur_set_);
        times_.resample_launches += 2;
    }
    cur_set_ = other;
    return LAMA_OK;
}

bool Engine::has_parked(int particle) const
{
    if (particle < 0) return d_->parked(cur_set_) != 0;
    if (particle >= cfg_.particles) return false;
    for (int k = 0; k < d_->view.n_kinds; ++k)
        if (d_->park_ol[cur_set_][(size_t)particle * d_->view.n_kinds + k].y) return true;
    return false;
}

Engine::WindowInfo Engine::window_info() const
{
    return WindowInfo{window_, d_->shifts, (uint64_t)d_->parked(cur_set_), d_->restored};
}

int Engine::shift_window(int32_t base_px, int32_t base_py)
{
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }   // ordered after the pending map update
    if (base_px == window_.base_px && base_py == window_.base_py) return LAMA_OK;
    const int32_t dim = window_.dim, max_patch = (int32_t)(0xFFFFFFFFu >> kPatchLog2) + 1 - dim;
    if (base_px < 0 || base_py < 0 || base_px > max_patch || base_py > max_patch) return fail("shift_window: window base outside the map's cell range", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const int set = cur_set_, n_lists = d_->n_lists();
    const DirWindow nw{base_px, base_py, dim};
    // scratch: counts | new {offset, length} | enter prefixes (window_shift_core.h: the arena may have gaps after a prune)
    const size_t b_cnt = (size_t)n_lists * sizeof(int2);
    const size_t b_enter = shift_scratch_ints(reinterpret_cast<const int32_t*>(d_->park_ol[set].data()), n_lists) * 4;
    if (d_->d_shift_scratch.reserve(2 * b_cnt + b_enter) != cudaSuccess) return fail("shift_window: out of device memory", LAMA_ERR_CUDA);
    int2* d_cnt = (int2*)d_->d_shift_scratch.get();
    int2* d_new_ol = d_cnt + n_lists;
    int32_t* d_enter = (int32_t*)(d_new_ol + n_lists);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    launch_shift_count(d_->view, d_->pv(set), set, nw, d_cnt, n_lists, d_->stream);
    CU_TRY(cudaGetLastError());
    std::vector<int2> cnt((size_t)n_lists), nol((size_t)n_lists);
    CU_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, b_cnt, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    int64_t total = 0, entered = 0;
    for (int i = 0; i < n_lists; ++i) {
        nol[i] = make_int2((int32_t)total, cnt[i].x);
        total += cnt[i].x;
        entered += cnt[i].y;
    }
    if (total > INT32_MAX) return fail("shift_window: too many parked entries", LAMA_ERR_POOL);
    DeviceArray<ParkEntry> arena;
    if (total) CU_TRY(arena.alloc((size_t)total));
    cudaError_t e = cudaMemcpyAsync(d_new_ol, nol.data(), b_cnt, cudaMemcpyHostToDevice, d_->stream);
    if (e == cudaSuccess) e = launch_shift_apply(d_->view, d_->pv(set), set, nw, arena.get(), d_new_ol, d_enter, n_lists, d_->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_->d_park_ol[set].get(), d_new_ol, b_cnt, cudaMemcpyDeviceToDevice, d_->stream);
    if (timing_ && e == cudaSuccess) e = cudaEventRecord(d_->ev[1], d_->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d_->stream);
    if (e != cudaSuccess) return fail(std::string("shift_window: ") + cudaGetErrorString(e), LAMA_ERR_CUDA);
    if (timing_) {
        float ms = 0;
        cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]);
        times_.shift_ms += ms;
    }
    d_->park[set] = std::move(arena);
    d_->park_ol[set] = nol;
    window_ = nw;
    d_->view.window = nw;
    d_->shifts += 1;
    d_->restored += (uint64_t)entered;
    times_.misc_launches += 2;
    return LAMA_OK;
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
    extent_stale_ = true;
    for (int k = 0; k < n_scans; ++k)
        if (offsets[k + 1] < offsets[k]) return fail("render_scans: offsets must not decrease", LAMA_ERR_ARG);
    const int64_t n_pts = offsets[n_scans];
    if (n_pts && !pts) return fail("render_scans: null points", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    std::vector<MovingTf> moving((size_t)n_scans);
    for (int k = 0; k < n_scans; ++k) moving[k] = moving_tf(origins ? origins + 3 * (size_t)k : nullptr, quats ? quats + 4 * (size_t)k : nullptr);
    // the groups and their windows, every scan checked before anything is written (render_plan.h); without following, one group in the
    // current window, whose kernels report a beam outside it
    std::vector<RenderGroup> groups;
    if (follow_) {
        std::vector<CellBox> boxes((size_t)n_scans);
        for (int k = 0; k < n_scans; ++k)
            boxes[k] = render_scan_box(compose_tf(states[k], moving[k]), 1.0 / cfg_.resolution, pts + 3 * offsets[k], offsets[k + 1] - offsets[k]);
        const int bad = plan_render(window_, boxes.data(), n_scans, groups);
        if (bad >= 0)
            return fail("render_scans: scan " + std::to_string(bad) + " reaches over more than one directory window (" + std::to_string(cfg_.dir_dim) +
                            " x " + std::to_string(cfg_.dir_dim) + " patches)",
                        LAMA_ERR_WINDOW);
    } else {
        groups.push_back(RenderGroup{0, n_scans, window_});
    }
    // scratch: points | offsets | moving | states | marks (dim^2 bytes) | cell counter
    auto up = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t dim2 = (size_t)cfg_.dir_dim * cfg_.dir_dim;
    const size_t b_pts = up((size_t)n_pts * 24), b_off = up((size_t)(n_scans + 1) * 8), b_mov = up((size_t)n_scans * sizeof(MovingTf)),
                 b_st = up((size_t)n_scans * sizeof(SE2)), b_marks = up(dim2);
    if (d_->d_scratch.reserve(b_pts + b_off + b_mov + b_st + b_marks + 16) != cudaSuccess) return fail("render_scans: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch.get();
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
    // The cell counters are sums, so the grouping changes no cell; `known` is ORed per group; the cell count adds up over the groups.
    float ms = 0.f;
    bool timed = false;
    for (const RenderGroup& g : groups) {
        if (g.window.base_px != window_.base_px || g.window.base_py != window_.base_py) {
            const int rc = shift_window(g.window.base_px, g.window.base_py);   // parked patches the window covers return before the marks
            if (rc != LAMA_OK) return rc;
        }
        if (grow_) {
            // every slot of a one-particle render-only map is one directory entry or one parked entry, so a group, which can fill at most
            // the empty entries of its window, always has room when the pool holds the parked entries and a whole window: no read-back
            const int64_t n_slots = d_->view.n_slots, want = pool_growth(n_slots, (int64_t)d_->parked(cur_set_), (int64_t)dim2, true);
            if (want != n_slots) {
                const int rc = grow_pool((int)want);
                if (rc != LAMA_OK) return rc;
            }
        }
        if (timed) {   // the previous group: every later group opens with a shift, which has synchronised the stream since
            float g_ms = 0.f;
            CU_TRY(cudaEventSynchronize(d_->ev_render[1]));
            CU_TRY(cudaEventElapsedTime(&g_ms, d_->ev_render[0], d_->ev_render[1]));
            ms += g_ms;
            timed = false;
        }
        RenderParams q = p;
        q.offsets += g.first;
        q.moving += g.first;
        q.states += g.first;
        if (timing_) CU_TRY(cudaEventRecord(d_->ev_render[0], d_->stream));
        launch_render_scans(d_->view, cur_set_, q, g.count, d_->stream);
        CU_TRY(cudaGetLastError());
        if (timing_) {
            CU_TRY(cudaEventRecord(d_->ev_render[1], d_->stream));
            timed = true;
        }
        times_.raycast_launches += 4;
    }
    unsigned long long n_cells = 0;
    CU_TRY(cudaMemcpyAsync(&n_cells, p.cells, 8, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timed) {
        float g_ms = 0.f;
        CU_TRY(cudaEventElapsedTime(&g_ms, d_->ev_render[0], d_->ev_render[1]));
        ms += g_ms;
    }
    times_.raycast_ms += ms;
    if (cells) *cells = n_cells;
    return check_device_status();
}

int Engine::pool_info(uint64_t out[2])
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    CU_TRY(cudaSetDevice(cfg_.device));
    int32_t free_count = 0;
    CU_TRY(cudaMemcpyAsync(&free_count, d_->view.free_count, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    out[0] = (uint64_t)d_->view.n_slots;
    out[1] = (uint64_t)(d_->view.n_slots - free_count);
    return LAMA_OK;
}

int Engine::grow_pool(int new_slots)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    StoreView& v = d_->view;
    if (cfg_.particles != 1) return fail("grow_pool: only a one-particle engine's pool grows", LAMA_ERR_STATE);
    if (new_slots <= v.n_slots) return LAMA_OK;
    if ((int64_t)new_slots > kPoolSlotCap) return fail("grow_pool: more than 2^24 - 2 slots (the slot field of a directory entry)", LAMA_ERR_POOL);
    CU_TRY(cudaSetDevice(cfg_.device));
    int32_t counts[2] = {0, 0};   // free, freed (released slots not yet merged)
    CU_TRY(cudaMemcpyAsync(counts, v.free_count, 8, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    const size_t n_old = (size_t)v.n_slots, n_new = (size_t)new_slots, n_add = n_new - n_old;
    // everything is allocated before anything is changed
    DeviceArray<char> pool_raw;
    DeviceArray<uint32_t> fbits, kbits;
    DeviceArray<int32_t> refcount, free_slots, freed;
    const bool ok = pool_raw.alloc((n_new + 1) * kPatchBytes) == cudaSuccess && fbits.alloc(n_new * 32) == cudaSuccess &&
                    (!v.kbits || kbits.alloc(n_new * 32) == cudaSuccess) && refcount.alloc(n_new) == cudaSuccess &&
                    free_slots.alloc(n_new) == cudaSuccess && freed.alloc(n_new) == cudaSuccess;
    auto give_up = [&](const std::string& why) {   // the new arrays are released on return, once the stream has passed them
        cudaStreamSynchronize(d_->stream);
        cudaGetLastError();   // a failed cudaMalloc is not sticky; clear it for the next call
        return fail("grow_pool: " + why + " (the pool keeps its " + std::to_string(n_old) + " slots)", LAMA_ERR_CUDA);
    };
    if (!ok) return give_up("out of device memory for " + std::to_string(n_new) + " slots");
    StoreView nv = v;
    nv.pool = reinterpret_cast<uint32_t*>(((uintptr_t)pool_raw.get() + (kPatchBytes - 1)) & ~(uintptr_t)(kPatchBytes - 1));
    nv.fbits = fbits.get();
    nv.kbits = kbits.get();
    nv.refcount = refcount.get();
    nv.free_slots = free_slots.get();
    nv.freed = freed.get();
    nv.n_slots = new_slots;
    // slots keep their ids; the free stack gets the new slots below the old free entries, the lowest new slot deepest of them, so the
    // old free slots are handed out first, then n_old, n_old + 1, ...
    cudaError_t e = cudaMemcpyAsync(nv.pool, v.pool, n_old * kPatchBytes, cudaMemcpyDeviceToDevice, d_->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nv.fbits, v.fbits, n_old * 128, cudaMemcpyDeviceToDevice, d_->stream);
    if (e == cudaSuccess && v.kbits) e = cudaMemcpyAsync(nv.kbits, v.kbits, n_old * 128, cudaMemcpyDeviceToDevice, d_->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nv.refcount, v.refcount, n_old * 4, cudaMemcpyDeviceToDevice, d_->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(nv.refcount + n_old, 0, n_add * 4, d_->stream);
    if (e == cudaSuccess) e = launch_fill_descending(nv.free_slots, (int)n_add, new_slots - 1, d_->stream);
    if (e == cudaSuccess && counts[0] > 0)
        e = cudaMemcpyAsync(nv.free_slots + n_add, v.free_slots, (size_t)counts[0] * 4, cudaMemcpyDeviceToDevice, d_->stream);
    if (e == cudaSuccess && counts[1] > 0) e = cudaMemcpyAsync(nv.freed, v.freed, (size_t)counts[1] * 4, cudaMemcpyDeviceToDevice, d_->stream);
    counts[0] += (int32_t)n_add;
    if (e == cudaSuccess) e = cudaMemcpyAsync(v.free_count, counts, 4, cudaMemcpyHostToDevice, d_->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d_->stream);
    if (e != cudaSuccess) return give_up(cudaGetErrorString(e));   // the old arrays are untouched; only the free count is written in place, last
    d_->pool_raw = std::move(pool_raw);
    d_->fbits = std::move(fbits);
    d_->kbits = std::move(kbits);
    d_->refcount = std::move(refcount);
    d_->free_slots = std::move(free_slots);
    d_->freed = std::move(freed);
    v = nv;
    cfg_.pool_slots = new_slots;
    pool_growths_ += 1;
    times_.misc_launches += 1;
    return LAMA_OK;
}

int Engine::prune_frequency()
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (!d_->view.kbits || cfg_.occupancy_kind != 0) return fail("prune_frequency: needs a frequency map with a known plane", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    extent_stale_ = true;
    launch_prune_freq(d_->view, cur_set_, d_->stream);
    const int n_parked = d_->park_ol[cur_set_][kMapOcc].y;   // particle 0's occupancy list
    if (n_parked) launch_prune_freq_parked(d_->view, d_->pv(cur_set_), n_parked, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += n_parked ? 2 : 1;
    return check_device_status();
}

int Engine::dm_apply(int particle, const uint32_t* cells_xy, const uint8_t* is_add, int n, uint32_t* processed)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || n < 0) return fail("dm_apply: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    uint32_t total = 0;
    const int cap = d_->ray.event_cap;
    // A following map runs each chunk's brushfire in a window that holds every cell it touches (dm_follow.h); every chunk is checked
    // before the first brushfire.  A fixed map runs every chunk in its window and refuses a cell outside it.
    std::vector<CellBox> boxes;
    std::vector<RenderGroup> groups;
    if (follow_ && n > 0) {
        const uint32_t reach = brushfire_reach((uint32_t)std::lround(std::sqrt((double)max_sqdist_)));
        const int bad = plan_dm_chunks(window_, cells_xy, n, cap, reach, boxes, groups);
        if (bad >= 0)
            return fail("dm_apply: cells " + std::to_string((int64_t)bad * cap) + " .. " + std::to_string(std::min<int64_t>(((int64_t)bad + 1) * cap, n) - 1) +
                            " of the list, grown by the brushfire's reach of " + std::to_string(reach) + " cells, span more than one directory window (" +
                            std::to_string(cfg_.dir_dim) + " x " + std::to_string(cfg_.dir_dim) + " patches)",
                        LAMA_ERR_WINDOW);
    }
    extent_stale_ = true;
    std::vector<uint64_t> ev;
    int done = 0;
    size_t g = 0;
    do {  // One brushfire over the whole list reproduces the reference (all cells queued, then ONE update()).  Lists longer than the
          // per-particle event buffer (2 048 cells) are applied in pieces with a brushfire after each, which gives a valid distance map but not necessarily the
          // reference's tie order -- big maps are loaded with lama_dm_read / lama_dm_import instead (DESIGN.md 10).
        int m = std::min(cap, n - done);
        if (!groups.empty()) {   // following: this chunk's window and, with a growing pool, a slot for every patch of its box
            const int chunk = done / cap;
            while (chunk >= groups[g].first + groups[g].count) ++g;
            const DirWindow& w = groups[g].window;
            if (w.base_px != window_.base_px || w.base_py != window_.base_py) {
                const int rc = shift_window(w.base_px, w.base_py);
                if (rc != LAMA_OK) return rc;
            }
            if (grow_) {
                uint64_t pool[2];
                int rc = pool_info(pool);
                const int64_t want = pool_growth((int64_t)pool[0], (int64_t)pool[1], box_patches(boxes[(size_t)chunk]), true);
                if (rc == LAMA_OK && want != (int64_t)pool[0]) rc = grow_pool((int)want);
                if (rc != LAMA_OK) return rc;
            }
        }
        ev.resize((size_t)std::max(m, 1));
        for (int i = 0; i < m; ++i) {
            uint32_t x = cells_xy[2 * (done + i)], y = cells_xy[2 * (done + i) + 1];
            if (dir_index(window_, x, y) < 0) return fail("dm_apply: cell outside the directory window", LAMA_ERR_WINDOW);
            ev[i] = push_record(((uint32_t)i << 1) | (is_add[done + i] ? 1u : 0u), cell_key(window_, x, y));
        }
        MapUpdateStats st{};
        st.events = (uint32_t)m;
        uint64_t* dev_ev = d_->d_events.get() + (size_t)particle * cap;
        CU_TRY(cudaMemcpyAsync(dev_ev, ev.data(), (size_t)m * 8, cudaMemcpyHostToDevice, d_->stream));
        CU_TRY(cudaMemcpyAsync(d_->d_stats.get() + particle, &st, sizeof(st), cudaMemcpyHostToDevice, d_->stream));
        const BrushParams bp = map_update_params(0, particle, nullptr);
        // block 0 of this launch must read the event list / stats of `particle`
        launch_brushfire(d_->view, bp, dev_ev, d_->d_stats.get() + particle, 1, d_->stream);
        launch_merge_free(d_->view, d_->stream);
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(d_->h_stats.get(), d_->d_stats.get() + particle, sizeof(MapUpdateStats), cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));
        times_.brushfire_launches += 1;
        times_.misc_launches += 1;
        total += d_->h_stats.get()[0].dm_pops;
        done += m;
        int rc = check_device_status();
        if (rc != LAMA_OK) return rc;
    } while (done < n);
    if (processed) *processed = total;
    return LAMA_OK;
}

// The dense directory of match_extent and match_fleet, built when a call allocated or deleted patches since the last one
int Engine::ensure_extent()
{
    if (!extent_stale_) return LAMA_OK;   // a shift moves entries between the window and the parked list, never between slots: it keeps the directory
    uint32_t mn[2], mx[2];
    const int n_patches = bounds(0, kMapDm, mn, mx);
    if (n_patches < 0) return fail("match_extent: reading the map's bounds failed", LAMA_ERR_CUDA);
    DirWindow xw{0, 0, 0};   // dim 0: no patch, every cell reads as absent
    if (extent_window(mn, mx, n_patches, &xw) < 0)
        return fail("match_extent: the map spans more than " + std::to_string(kExtentMaxPatches) + " patches on an axis", LAMA_ERR_WINDOW);
    if (xw.dim) {
        const size_t bytes = (size_t)xw.dim * xw.dim * 4;
        if (d_->d_extent.reserve(bytes) != cudaSuccess) return fail("match_extent: out of device memory", LAMA_ERR_CUDA);
        CU_TRY(cudaMemsetAsync(d_->d_extent.get(), 0xFF, bytes, d_->stream));
        launch_extent_dir(d_->view, d_->pv(cur_set_), cur_set_, xw, d_->park_ol[cur_set_][kMapDm].y, (int32_t*)d_->d_extent.get(), d_->stream);
        CU_TRY(cudaGetLastError());
        times_.misc_launches += 1;
    }
    extent_ = xw;
    extent_stale_ = false;
    return LAMA_OK;
}

int Engine::match_extent(const SE2* states, int count, const SolverOptions& so, double meas_sigma, HostMatchResult* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count < 1) return fail("match_extent: no states", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("match_extent: no scan uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    { int rc = ensure_extent(); if (rc != LAMA_OK) return rc; }
    MatchParams mp = match_params(so, meas_sigma, 0, true, 1);
    mp.parked_any = 0;   // k_match_extent reads parked patches through its directory: no read sets kErrWindow
    return match_sync(states, count, mp, true, out);
}

int Engine::fleet_reserve(int robots, const double* offsets_xy, int n_off)
{
    if (d_->d_fleet) return fail("fleet_reserve: already reserved", LAMA_ERR_STATE);
    if (robots < 1 || n_off < 1 || !offsets_xy) return fail("fleet_reserve: bad arguments", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    const size_t bytes = (size_t)robots * (sizeof(FleetScan) + (size_t)cfg_.max_beams * 24);
    CU_TRY(d_->d_fleet.alloc(bytes));
    CU_TRY(d_->h_fleet.alloc(bytes));
    CU_TRY(d_->d_fleet_off.alloc((size_t)n_off * 2));
    CU_TRY(d_->d_fleet_lik.alloc((size_t)robots * n_off));
    CU_TRY(d_->h_fleet_lik.alloc((size_t)robots * n_off));
    CU_TRY(cudaMemcpy(d_->d_fleet_off.get(), offsets_xy, (size_t)n_off * 16, cudaMemcpyHostToDevice));
    d_->fleet_cap = robots;
    d_->fleet_n_off = n_off;
    return LAMA_OK;
}

int Engine::fleet_scans(const double* pts, const int* n_points, int count, const double* origins, const double* quats)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count < 1 || count > d_->fleet_cap || !pts || !n_points) return fail("fleet_scans: bad arguments", LAMA_ERR_ARG);
    for (int k = 0; k < count; ++k)
        if (n_points[k] < 1 || n_points[k] > cfg_.max_beams) return fail("fleet_scans: number of beams out of range", LAMA_ERR_ARG);
    CU_TRY(cudaSetDevice(cfg_.device));
    FleetScan* desc = (FleetScan*)d_->h_fleet.get();
    double* hp = (double*)(d_->h_fleet.get() + (size_t)d_->fleet_cap * sizeof(FleetScan));
    int64_t off = 0;
    int max_n = 0;
    for (int k = 0; k < count; ++k) {
        desc[k] = FleetScan{off, n_points[k], 0, moving_tf(origins ? origins + 3 * k : nullptr, quats ? quats + 4 * k : nullptr)};
        off += n_points[k];
        max_n = std::max(max_n, n_points[k]);
    }
    std::memcpy(hp, pts, (size_t)off * 24);
    // descriptors and points in one copy: everything from the first descriptor to the last point
    const size_t bytes = (size_t)d_->fleet_cap * sizeof(FleetScan) + (size_t)off * 24;
    CU_TRY(cudaMemcpyAsync(d_->d_fleet.get(), d_->h_fleet.get(), bytes, cudaMemcpyHostToDevice, d_->stream));
    h2d_bytes_ += bytes;
    d_->fleet_max_beams = max_n;
    return LAMA_OK;
}

int Engine::match_fleet(const int32_t* scan_of_block, const SE2* states, int count, int mode, const SolverOptions& so, double meas_sigma)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (count < 1 || !scan_of_block || !states || (mode != 0 && mode != 1)) return fail("match_fleet: bad arguments", LAMA_ERR_ARG);
    if (d_->fleet_max_beams < 1) return fail("match_fleet: no fleet scans uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    const bool extent = follow_ && has_parked();
    if (extent) { int rc = ensure_extent(); if (rc != LAMA_OK) return rc; }
    if ((size_t)count > d_->h_fleet_blocks.size()) {   // h_fleet_blocks is allocated last
        d_->d_fleet_blocks.reset(); d_->h_fleet_blocks.reset();
        CU_TRY(d_->d_fleet_blocks.alloc((size_t)count));
        CU_TRY(d_->h_fleet_blocks.alloc((size_t)count));
    }
    std::memcpy(d_->h_fleet_blocks.get(), scan_of_block, (size_t)count * 4);
    CU_TRY(cudaMemcpyAsync(d_->d_fleet_blocks.get(), d_->h_fleet_blocks.get(), (size_t)count * 4, cudaMemcpyHostToDevice, d_->stream));
    { int rc = upload_states(states, count, d_->stream); if (rc != LAMA_OK) return rc; }
    MatchParams mp = match_params(so, meas_sigma, 0, true, mode);
    mp.points = d_->fleet_points();
    mp.scan.scale = 1.0 / cfg_.resolution;
    if (extent) mp.parked_any = 0;   // the dense directory holds the parked patches
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[0], d_->stream));
    launch_match_fleet(d_->view, mp, d_->fleet_scans(), d_->d_fleet_blocks.get(), d_->fleet_max_beams, extent ? (const int32_t*)d_->d_extent.get() : nullptr, extent_,
                       d_->d_states.get(), d_->d_results.get(), count, d_->stream);
    if (timing_) CU_TRY(cudaEventRecord(d_->ev[1], d_->stream));
    CU_TRY(cudaGetLastError());
    times_.match_launches += 1;
    fleet_count_ = count;
    fleet_parked_ = mp.parked_any != 0;
    fleet_sampled_ = false;
    return LAMA_OK;
}

int Engine::sampling_fleet()
{
    if (fleet_count_ < 1 || fleet_count_ > d_->fleet_cap) return fail("sampling_fleet: no fleet match of at most one block per robot", LAMA_ERR_STATE);
    launch_sampling_fleet(d_->view, d_->pv(cur_set_), cur_set_, d_->fleet_points(), d_->fleet_scans(), d_->d_fleet_blocks.get(), d_->d_results.get(), fleet_count_,
                          1.0 / cfg_.resolution, d_->d_fleet_off.get(), d_->fleet_n_off, cfg_.resolution, max_sqdist_, d_->d_fleet_lik.get(), d_->stream);
    CU_TRY(cudaGetLastError());
    times_.misc_launches += 1;
    fleet_sampled_ = true;
    return LAMA_OK;
}

int Engine::fleet_results(HostMatchResult* out, double* lik)
{
    const int count = fleet_count_;
    if (count < 1) return fail("fleet_results: no fleet match", LAMA_ERR_STATE);
    fleet_count_ = 0;
    CU_TRY(cudaMemcpyAsync(d_->h_results.get(), d_->d_results.get(), (size_t)count * sizeof(MatchResult), cudaMemcpyDeviceToHost, d_->stream));
    const size_t lik_n = fleet_sampled_ ? (size_t)count * d_->fleet_n_off : 0;
    if (lik_n) CU_TRY(cudaMemcpyAsync(d_->h_fleet_lik.get(), d_->d_fleet_lik.get(), lik_n * 8, cudaMemcpyDeviceToHost, d_->stream));
    if (fleet_parked_) CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (timing_) {
        float ms = 0;
        cudaEventElapsedTime(&ms, d_->ev[0], d_->ev[1]);
        times_.match_ms += ms;
    }
    if (fleet_parked_ && *d_->h_status.get()) return check_device_status();
    std::memcpy(out, d_->h_results.get(), (size_t)count * sizeof(MatchResult));
    if (lik && lik_n) std::memcpy(lik, d_->h_fleet_lik.get(), lik_n * 8);
    d2h_bytes_ += (uint64_t)count * sizeof(MatchResult) + lik_n * 8;
    return LAMA_OK;
}

int Engine::sampling_likelihood(int particle, const SE2& pose, const double* offsets_xy, int n, int stride, double* out)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles || n < 1 || stride < 1) return fail("sampling_likelihood: bad arguments", LAMA_ERR_ARG);
    if (d_->scan.n_beams < 1) return fail("sampling_likelihood: no scan uploaded", LAMA_ERR_STATE);
    CU_TRY(cudaSetDevice(cfg_.device));
    if (d_->d_scratch.reserve((size_t)n * 24) != cudaSuccess) return fail("sampling_likelihood: out of device memory", LAMA_ERR_CUDA);
    double* d_off = (double*)d_->d_scratch.get();
    double* d_out = d_off + 2 * (size_t)n;
    CU_TRY(cudaMemcpyAsync(d_off, offsets_xy, (size_t)n * 16, cudaMemcpyHostToDevice, d_->stream));
    launch_sampling(d_->view, d_->pv(cur_set_), cur_set_, particle, d_->d_points, d_->scan, pose, d_off, n, stride, cfg_.resolution, max_sqdist_, d_out, d_->stream);
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
    if (d_->d_scratch.reserve(bp + bd + bg) != cudaSuccess) return fail("dm_distance: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch.get();
    CU_TRY(cudaMemcpyAsync(base, pts, bp, cudaMemcpyHostToDevice, d_->stream));
    launch_distance(d_->view, d_->pv(cur_set_), cur_set_, particle, (const double*)base, n, cfg_.resolution, max_sqdist_, (double*)(base + bp),
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
    if (d_->d_scratch.reserve(bw + bpz) != cudaSuccess) return fail("export_window: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch.get();
    launch_export(d_->view, d_->pv(cur_set_), cur_set_, particle, kind, x0, y0, w, h, (uint32_t*)base, (uint8_t*)(base + bw), d_->stream);
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
    if (d_->d_scratch.reserve(bc + bw + bf) != cudaSuccess) return fail("gather_cells: out of device memory", LAMA_ERR_CUDA);
    char* base = (char*)d_->d_scratch.get();
    CU_TRY(cudaMemcpyAsync(base, cells_xy, bc, cudaMemcpyHostToDevice, d_->stream));
    launch_gather_cells(d_->view, d_->pv(cur_set_), cur_set_, particle, kind, (const uint32_t*)base, n, (uint32_t*)(base + bc), (uint8_t*)(base + bc + bw), d_->stream);
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
    if (d_->d_scratch.reserve((size_t)w * h) != cudaSuccess) return fail("export_bits: out of device memory", LAMA_ERR_CUDA);
    launch_export_bits(d_->view, d_->pv(cur_set_), plane, cur_set_, particle, x0, y0, w, h, (uint8_t*)d_->d_scratch.get(), d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, d_->d_scratch.get(), (size_t)w * h, cudaMemcpyDeviceToHost, d_->stream));
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
    extent_stale_ = true;
    const size_t bw = (size_t)w * h * 4;
    if (d_->d_scratch.reserve(bw) != cudaSuccess) return fail("import_window: out of device memory", LAMA_ERR_CUDA);
    CU_TRY(cudaMemcpyAsync(d_->d_scratch.get(), words, bw, cudaMemcpyHostToDevice, d_->stream));
    launch_import(d_->view, cur_set_, particle, kind, x0, y0, w, h, (const uint32_t*)d_->d_scratch.get(), d_->stream);
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
    CU_TRY(cudaStreamSynchronize(d_->stream));
    times_.misc_launches += 2;
    return check_device_status();
}

static const uint32_t kPackMagic = 0x4c414d50u;  // "LAMP"

int Engine::pack_size(int particle, size_t* bytes)
{
    { int rc_settle = settle(nullptr); if (rc_settle != LAMA_OK) return rc_settle; }
    if (particle < 0 || particle >= cfg_.particles) return fail("pack_size: bad particle", LAMA_ERR_ARG);
    if (has_parked(particle)) return fail("pack: the particle's maps have parked entries (the window has moved), which a blob does not carry", LAMA_ERR_STATE);
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
    while (d_->mig_chunk < d_->mig_chunks.size() && d_->mig_off + need > d_->mig_chunks[d_->mig_chunk].size()) {
        ++d_->mig_chunk;
        d_->mig_off = 0;
    }
    if (d_->mig_chunk == d_->mig_chunks.size()) {
        const size_t chunk = std::max(need, (size_t)64 << 20);
        DeviceArray<char> c;
        CU_TRY(c.alloc(chunk));
        d_->mig_chunks.push_back(std::move(c));
        d_->mig_off = 0;
    }
    *dptr = d_->mig_chunks[d_->mig_chunk].get() + d_->mig_off;
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
    if (has_parked(particle)) return fail("pack: the particle's maps have parked entries (the window has moved), which a blob does not carry", LAMA_ERR_STATE);
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
    extent_stale_ = true;
    const size_t n = (size_t)blob.n_occ + blob.n_dm, ne = blob_entry_bytes(n);
    if (particle < 0 || particle >= cfg_.particles || blob.bytes < ne + n * (size_t)(kPatchBytes + 128)) return fail("unpack: bad arguments", LAMA_ERR_ARG);
    if (has_parked(particle)) return fail("unpack: the slot's maps have parked entries (the window has moved)", LAMA_ERR_STATE);
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
    CU_TRY(cudaMemcpyAsync(d_->h_status.get(), d_->view.status, 4, cudaMemcpyDeviceToHost, d_->stream));
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
    extent_stale_ = true;
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
    extent_stale_ = true;
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
    // parked patches: the same test; each list keeps its offset and shrinks to the entries that stay
    const int nk = d_->view.n_kinds;
    std::vector<int32_t> dropped;                       // their directory entries, one reference each
    std::vector<std::pair<int32_t, int32_t>> gone;      // patch coordinates removed from kinds 0 / 1 (counted once per patch)
    for (int k = 0; k < nk; ++k) {
        const size_t li = (size_t)particle * nk + k;
        const int2 ol = d_->park_ol[cur_set_][li];
        if (ol.y == 0) continue;
        std::vector<ParkEntry> l((size_t)ol.y), keep;
        CU_TRY(cudaMemcpyAsync(l.data(), d_->park[cur_set_].get() + ol.x, l.size() * sizeof(ParkEntry), cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));
        for (const ParkEntry& e : l) {
            const uint32_t c0[2] = {(uint32_t)e.px << kPatchLog2, (uint32_t)e.py << kPatchLog2};
            bool meets = true;
            for (int a = 0; a < 2; ++a) {
                const double ws = ((double)c0[a] - off) / scale, we = ((double)(c0[a] + kPatchLen) - off) / scale;
                const double bh = (we - ws) * 0.5, bc = ws + bh;
                meets = meets && (std::abs(center[a] - bc) <= (hwidth[a] + bh));
            }
            if (meets) {
                keep.push_back(e);
            } else {
                dropped.push_back(e.entry);
                if (k < 2) gone.push_back({e.py, e.px});
            }
        }
        if (keep.size() == l.size()) continue;
        if (!keep.empty())
            CU_TRY(cudaMemcpyAsync(d_->park[cur_set_].get() + ol.x, keep.data(), keep.size() * sizeof(ParkEntry), cudaMemcpyHostToDevice, d_->stream));
        d_->park_ol[cur_set_][li].y = (int32_t)keep.size();
        CU_TRY(cudaMemcpyAsync(d_->d_park_ol[cur_set_].get() + li, &d_->park_ol[cur_set_][li], sizeof(int2), cudaMemcpyHostToDevice, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));   // `keep` and the host list entry are read by the copies
    }
    std::sort(gone.begin(), gone.end());
    const size_t n_gone = (size_t)(std::unique(gone.begin(), gone.end()) - gone.begin());
    if (removed) *removed = (int)(list.size() + n_gone);
    if (list.empty() && dropped.empty()) return LAMA_OK;
    if (!list.empty()) {
        std::memcpy(d_->h_idx.get(), list.data(), list.size() * 4);
        CU_TRY(cudaMemcpyAsync(d_->d_idx.get(), d_->h_idx.get(), list.size() * 4, cudaMemcpyHostToDevice, d_->stream));
        launch_delete_patches(d_->view, cur_set_, particle, d_->d_idx.get(), (int)list.size(), d_->stream);
    }
    if (!dropped.empty()) {
        if (d_->d_scratch.reserve(dropped.size() * 4) != cudaSuccess) return fail("prune_outside: out of device memory", LAMA_ERR_CUDA);
        CU_TRY(cudaMemcpyAsync(d_->d_scratch.get(), dropped.data(), dropped.size() * 4, cudaMemcpyHostToDevice, d_->stream));
        launch_release_entries(d_->view, (const int32_t*)d_->d_scratch.get(), (int)dropped.size(), d_->stream);
    }
    launch_merge_free(d_->view, d_->stream);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaStreamSynchronize(d_->stream));
    if (d_->parked(cur_set_) == 0 && d_->park[cur_set_]) d_->drop_arena(cur_set_);
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
    std::vector<ParkEntry> l;
    if (d_->fetch(cur_set_, (size_t)particle * d_->view.n_kinds + kind, l) != cudaSuccess) return -1;
    for (const ParkEntry& e : l) {
        const uint32_t x = (uint32_t)e.px << kPatchLog2, y = (uint32_t)e.py << kPatchLog2;
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
        // parked patches, by the same rule: the two lists are sorted by patch, so walk them side by side
        std::vector<ParkEntry> lk, lo;
        if (d_->fetch(cur_set_, (size_t)p * d_->view.n_kinds + kind, lk) != cudaSuccess) return -1;
        if (kind == 1 && d_->fetch(cur_set_, (size_t)p * d_->view.n_kinds, lo) != cudaSuccess) return -1;
        size_t i = 0, j = 0;
        while (i < lk.size() || j < lo.size()) {
            const ParkEntry* a = i < lk.size() ? &lk[i] : nullptr;
            const ParkEntry* b = j < lo.size() ? &lo[j] : nullptr;
            const bool take_a = a && (!b || !park_before(b->px, b->py, a->px, a->py));
            const bool take_b = b && (!a || !park_before(a->px, a->py, b->px, b->py));
            const int ud = take_a ? ref[(size_t)(a->entry & kDirSlotMask)] : 0, uo = take_b ? ref[(size_t)(b->entry & kDirSlotMask)] : 0;
            i += take_a;
            j += take_b;
            const int uses = kind == 0 ? ud : (ud > 0 && uo > 0 ? std::min(ud, uo) : std::max(ud, uo));
            if (uses <= 0 && kind == 1) continue;
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
struct PinnedPair {   // two pinned chunk buffers and their completion events: no buffer goes while a copy may still use it
    PinnedArray<char> buf[2];
    Event done[2];
    cudaError_t init()
    {
        for (int b = 0; b < 2; ++b) {
            cudaError_t e = buf[b].alloc(kCkptChunk);
            if (e == cudaSuccess) e = done[b].create(cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    ~PinnedPair()
    {
        for (const Event& d : done)
            if (d) cudaEventSynchronize(d);
    }
};
double host_ms(std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); }
}  // namespace

int Engine::snapshot(EngineImage* out, CheckpointTimes* t, int particles)
{
    if (particles == 0) particles = cfg_.particles;
    if (particles < 0 || particles > cfg_.particles) return fail("snapshot: particle count out of range", LAMA_ERR_ARG);
    { int rc = settle(nullptr); if (rc != LAMA_OK) return rc; }
    CU_TRY(cudaSetDevice(cfg_.device));
    const StoreView& v = d_->view;
    const size_t n_slots = (size_t)v.n_slots, n_dir = (size_t)particles * v.n_kinds * cfg_.dir_dim * cfg_.dir_dim;
    DeviceArray<int32_t> d_cnt, d_used, d_new_id, d_list, d_ref, d_dirs, d_parked_in, d_parked_out;
    DeviceArray<uint32_t> d_bad;
    DeviceArray<char> d_temp, d_stage;
    CkptScratch c{};
    c.temp_bytes = ckpt_scan_temp_bytes(v.n_slots);
    CU_TRY(d_cnt.alloc(n_slots));
    CU_TRY(d_used.alloc(n_slots));
    CU_TRY(d_new_id.alloc(n_slots));
    CU_TRY(d_list.alloc(n_slots));
    CU_TRY(d_ref.alloc(n_slots));
    CU_TRY(d_dirs.alloc(n_dir));
    CU_TRY(d_bad.alloc(4));
    CU_TRY(d_temp.alloc(std::max<size_t>(c.temp_bytes, 16)));
    c.cnt = d_cnt.get(); c.used = d_used.get(); c.new_id = d_new_id.get(); c.list = d_list.get(); c.ref = d_ref.get(); c.dirs = d_dirs.get();
    c.bad = d_bad.get(); c.temp = d_temp.get();
    // the parked entries of the saved particles, gathered list by list in (particle, kind) order; counted and remapped with the directories
    std::vector<int32_t> park_len((size_t)particles * v.n_kinds, 0);
    std::vector<ParkEntry> parked;
    for (size_t li = 0; li < park_len.size(); ++li) {
        std::vector<ParkEntry> l;
        CU_TRY(d_->fetch(cur_set_, li, l));
        park_len[li] = (int32_t)l.size();
        parked.insert(parked.end(), l.begin(), l.end());
    }
    std::vector<int32_t> park_entries(parked.size());
    for (size_t i = 0; i < parked.size(); ++i) park_entries[i] = parked[i].entry;
    c.n_parked = parked.size();
    c.parked = nullptr;
    c.parked_out = nullptr;
    if (c.n_parked) {
        CU_TRY(d_parked_in.alloc(c.n_parked));
        CU_TRY(d_parked_out.alloc(c.n_parked));
        CU_TRY(cudaMemcpyAsync(d_parked_in.get(), park_entries.data(), c.n_parked * 4, cudaMemcpyHostToDevice, d_->stream));
        c.parked = d_parked_in.get();
        c.parked_out = d_parked_out.get();
    }
    Event ev[4];
    for (Event& x : ev) CU_TRY(x.create(cudaEventDefault));
    CU_TRY(cudaMemsetAsync(c.cnt, 0, n_slots * 4, d_->stream));
    CU_TRY(cudaMemsetAsync(c.bad, 0, 4, d_->stream));
    CU_TRY(cudaEventRecord(ev[0], d_->stream));
    launch_ckpt_compact(v, cur_set_, particles, c, d_->stream, ev[1]);
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
    img.particles = particles; img.dir_dim = cfg_.dir_dim; img.pool_slots = cfg_.pool_slots; img.max_beams = cfg_.max_beams;
    img.occupancy_kind = cfg_.occupancy_kind; img.known_plane = cfg_.known_plane; img.resolution = cfg_.resolution; img.l2_max = cfg_.l2_max;
    img.window = window_;
    img.used = K;
    img.park_len.clear();
    img.parked.clear();
    if (c.n_parked) {
        CU_TRY(cudaMemcpyAsync(park_entries.data(), c.parked_out, c.n_parked * 4, cudaMemcpyDeviceToHost, d_->stream));
        CU_TRY(cudaStreamSynchronize(d_->stream));
        for (size_t i = 0; i < parked.size(); ++i) parked[i].entry = park_entries[i];
        img.park_len = park_len;
        img.parked = parked;
    }
    const size_t stride = img.slot_stride(), bytes = (size_t)K * stride;
    CU_TRY(d_stage.alloc(std::max<size_t>(bytes, 16)));
    char* stage = d_stage.get();
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
            CU_TRY(cudaMemcpyAsync(pin.buf[i & 1].get(), stage + off, len, cudaMemcpyDeviceToHost, d_->stream));
            CU_TRY(cudaEventRecord(pin.done[i & 1], d_->stream));
        }
        if (i > 0) {
            const size_t j = i - 1, off = j * kCkptChunk, len = std::min(kCkptChunk, bytes - off);
            CU_TRY(cudaEventSynchronize(pin.done[j & 1]));
            std::memcpy(img.slot_store.data() + off, pin.buf[j & 1].get(), len);
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

Engine* Engine::restore(const EngineImage& img, int device, uint64_t stream, std::string& err, CheckpointTimes* t, int capacity)
{
    const auto t0 = std::chrono::steady_clock::now();
    if (capacity == 0) capacity = img.particles;
    if (capacity < img.particles) { err = "restore: capacity below the image's particles"; return nullptr; }
    EngineConfig cfg;
    cfg.device = device; cfg.particles = capacity; cfg.resolution = img.resolution; cfg.l2_max = img.l2_max; cfg.dir_dim = img.dir_dim;
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
    if (img.slot_src.empty()) {
        const size_t n_chunks = (bytes + kCkptChunk - 1) / kCkptChunk;
        for (size_t i = 0; i < n_chunks; ++i) {
            const size_t off = i * kCkptChunk, len = std::min(kCkptChunk, bytes - off);
            if (i >= 2 && !cu(cudaEventSynchronize(pin.done[i & 1]), "copy")) return nullptr;   // chunk i - 2 has left this buffer
            std::memcpy(pin.buf[i & 1].get(), img.slot_bytes + off, len);
            size_t base = 0;
            for (const Region& r : regions) {   // the chunk may straddle the cells and the planes
                const size_t lo = std::max(off, base), hi = std::min(off + len, base + r.len);
                if (lo < hi && !cu(cudaMemcpyAsync(r.dst + (lo - base), pin.buf[i & 1].get() + (lo - off), hi - lo, cudaMemcpyHostToDevice, d->stream), "copy"))
                    return nullptr;
                base += r.len;
            }
            if (!cu(cudaEventRecord(pin.done[i & 1], d->stream), "copy")) return nullptr;
        }
    } else {
        // the same byte stream (cells of slots 0 .. K-1, then their planes), assembled piece by piece from the listed slots; a piece
        // (4 KiB of cells or 128 B of bits) never straddles a chunk, since the chunk size is a multiple of both
        size_t i = 0, fill = 0;
        const int last_region = regions[2].len ? 2 : 1;
        for (int r = 0; r <= last_region; ++r) {
            const size_t piece = r == 0 ? (size_t)kPatchBytes : 128;
            for (uint32_t k = 0; k < K; ++k) {
                const EngineImage::SlotRef& s = img.slot_src[k];
                const size_t plane = r == 0 ? 0 : (size_t)s.count * (kPatchBytes + (r == 2 ? 128 : 0));
                if (fill == 0 && i >= 2 && !cu(cudaEventSynchronize(pin.done[i & 1]), "copy")) return nullptr;   // chunk i - 2 has left this buffer
                std::memcpy(pin.buf[i & 1].get() + fill, s.payload + plane + (size_t)s.slot * piece, piece);
                fill += piece;
                if (fill < kCkptChunk && !(r == last_region && k + 1 == K)) continue;
                const size_t off = i * kCkptChunk;
                size_t base = 0;
                for (const Region& g : regions) {
                    const size_t lo = std::max(off, base), hi = std::min(off + fill, base + g.len);
                    if (lo < hi && !cu(cudaMemcpyAsync(g.dst + (lo - base), pin.buf[i & 1].get() + (lo - off), hi - lo, cudaMemcpyHostToDevice, d->stream), "copy"))
                        return nullptr;
                    base += g.len;
                }
                if (!cu(cudaEventRecord(pin.done[i & 1], d->stream), "copy")) return nullptr;
                ++i;
                fill = 0;
            }
        }
    }
    // the parked lists into set 0's arena, in the image's order
    if (!img.parked.empty()) {
        std::vector<int2>& ol = d->park_ol[0];
        int32_t off = 0;
        for (size_t li = 0; li < img.park_len.size(); ++li) {
            ol[li] = make_int2(off, img.park_len[li]);
            off += img.park_len[li];
        }
        if (!cu(d->park[0].alloc(img.parked.size()), "parked entries") ||
            !cu(cudaMemcpyAsync(d->park[0].get(), img.parked.data(), img.parked.size() * sizeof(ParkEntry), cudaMemcpyHostToDevice, d->stream), "parked entries") ||
            !cu(cudaMemcpyAsync(d->d_park_ol[0].get(), ol.data(), ol.size() * sizeof(int2), cudaMemcpyHostToDevice, d->stream), "parked lists"))
            return nullptr;
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
